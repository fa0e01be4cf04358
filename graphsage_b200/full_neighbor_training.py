"""Whole-neighbourhood layers: SampleAndAggregate.full_neighbor_embeddings (contract: oracle/full_neighbor.py) and its
differentiable form, full-batch training (contract: oracle/full_neighbor_grad.py).

One layer implementation, _FullLayer, serves both.  Inference runs its forward under no_grad; training runs it as a
branch of supervised_models._LayerFn, the autograd Function of every aggregator, so the training forward is the
inference layer and the values are the same bits.  The backward:
  - weight gradients dW = X^T dZ as library matmuls, as in the sampled path (_LayerFn);
  - source gradients through the CSR kernels over the transposed graph (ops.csr_transpose, built once per CSR and cached
    on the model): the means' backward is ops.csr_aggregate(op="sum") of g / count, the max-pool's ops.csr_max_backward;
  - the last layer reads only the rows of node_ids (duplicates allowed): their gradients are scattered into a dense
    [N+1, w] gradient by ops.embedding_grad (group 1) first.
The pools run their MLP once per node, as full_neighbor_embeddings does, whatever fused_pool says: the MLP input is the
layer's whole [N+1, in] table, so its gradient dZ Wm^T needs no transpose.  Layer-0 feature columns are not trainable:
with identity_dim = 0 layer 0 computes no source gradient (the pools still compute dWm, dbm); with identity_dim = d > 0 it
computes columns [0, d) only, which autograd delivers as model.embeds.grad (a dense [N+1, d] tensor).

Minibatches (minibatch=True; contract: oracle/full_neighbor_blocks.py) run the same layers over the
seeds' receptive field: ops.csr_blocks builds one block per layer - a local CSR over V_l, the nodes layer l reads - and
layer l runs over its block with the block's rows, exactly as the whole-graph layers run over the whole CSR.  Layer 0
reads the global table: the means through the global CSR with rows = V_1, the pools' MLP on V_0's rows only (read by id,
ops.TableRows), reduced through block 0.  Same bits as the whole-graph pass for the seeds; every buffer is block-sized.
The blocks and their transposes are built per call, not cached.

Training dropout (dropout=p > 0; contract: oracle/full_neighbor_dropout.py) masks by global identities: per CSR entry for
the means' neighbour branch (gs_csr_aggregate_dropout, the entry's global CSR position), per node for the mean's self
rows, GCN's own row and the pools' MLP input (ops.dropout_apply by id).  Each graph carries the position map of its
kernels - (indptr, None, nnz) for the whole graph, (global indptr, src_ids, global nnz) for a block - so a block masks every
element as the whole-graph pass does.  The backward regenerates every mask: the transposed sum reads the transpose's
t_slot (ops.csr_transpose(slots=True)) to find each entry's forward position.
"""
import torch

from . import ops
from .aggregators import GCNAggregator, MaxPoolingAggregator, SeqAggregator, TwoMaxLayerPoolingAggregator, _rows
from .host_features import refuse_host_table
from .int8_features import refuse_int8_table
from .layers import act_code
from .supervised_models import (_LayerFn, build_aggregators, check_full_neighbor_dropout, full_neighbor_site_plan,
                                layer_params)


class FullNeighborGraph(object):
    """The transposes and divisors of one CSR, built on first use.  `key` identifies the CSR tensors (data_ptr, numel,
    _version of both); the tensors themselves are held, so their memory cannot be reused by a different CSR while cached."""

    def __init__(self, indptr, indices, pos_map=None):
        """pos_map: (pos_indptr, pos_ids or None, pos_nnz), how the masks name this CSR's rows and entries globally
        (default: the CSR is the global one)."""
        self.indptr, self.indices = indptr, indices
        self.pos_map = pos_map if pos_map is not None else (indptr, None, indices.numel())
        self.key = FullNeighborGraph.key_of(indptr, indices)
        self.n_rows = indptr.numel()                 # N + 1
        self._t, self._counts = {}, {}

    @staticmethod
    def key_of(indptr, indices):
        return tuple((t.data_ptr(), t.numel(), t._version) for t in (indptr, indices))

    def transpose(self, with_self, slots=False):
        """(t_indptr, t_indices), or with slots (t_indptr, t_indices, t_slot); a slotted transpose serves both."""
        if (with_self, True) in self._t:
            return self._t[(with_self, True)] if slots else self._t[(with_self, True)][:2]
        if slots:
            self._t.pop(with_self, None)
            self._t[(with_self, True)] = ops.csr_transpose(self.indptr, self.indices, with_self=with_self, slots=True)
            return self._t[(with_self, True)]
        if with_self not in self._t:
            self._t[with_self] = ops.csr_transpose(self.indptr, self.indices, with_self=with_self)
        return self._t[with_self]

    def counts(self, with_self):
        """The forward's divisors for the N + 1 effective rows (max(degree, 1), + 1 for GCN), fp32 [N + 1, 1]."""
        if with_self not in self._counts:
            deg = (self.indptr[1:] - self.indptr[:-1]).clamp(min=1)
            one = torch.ones((1,), dtype=deg.dtype, device=deg.device)
            self._counts[with_self] = (torch.cat([deg, one]) + int(with_self)).to(torch.float32).unsqueeze(1)
        return self._counts[with_self]

    def mean_backward(self, g, with_self, sites=None):
        """d(source) of the mean over the effective rows for their gradient g [N + 1, w]: sum of g / count over the
        transposed rows; sites = (neighbour, self): the forward's masks, regenerated through t_slot."""
        gp = (g / self.counts(with_self)).contiguous()
        if sites is None:
            t_indptr, t_indices = self.transpose(with_self)
            return ops.csr_aggregate(gp, t_indptr, t_indices, "sum")
        t_indptr, t_indices, t_slot = self.transpose(with_self, slots=True)
        return ops.csr_aggregate(gp, t_indptr, t_indices, "sum", dropout=(sites[0], sites[1], self.pos_map), t_slot=t_slot)

    def node_ids(self, rows):
        """The global node ids of local rows (None: every row) for the per-node masks; None when they are the rows."""
        ids = self.pos_map[1]
        if rows is None:
            return ids
        return rows if ids is None else ids.index_select(0, rows.long())


class _FullLayer(object):
    """One aggregator layer over a graph's rows, and the _LayerFn branch that trains it: rows None computes all of them,
    else the rows of `rows` (ids of the graph's nodes).  A block's layer 0 (src_ids = V_0's global ids) reads the global
    [N+1, .] table instead: its reductions of the table through table_csr = (global indptr, global indices, V_1's global
    ids), the pools' MLP on V_0's rows; everything after the MLP, and the whole backward, is in the graph's (block 0's)
    local space."""

    def __init__(self, agg, graph, rows, src_ids=None, table_csr=None):
        self.agg, self.graph, self.rows = agg, graph, rows
        self.src_ids, self.table_csr = src_ids, table_csr
        self.sites = None                       # training dropout: {"neigh", "self"} or {"mlp"} -> (seed, call, rate)
        self.gcn = isinstance(agg, GCNAggregator)
        self.pool = isinstance(agg, MaxPoolingAggregator)
        self.row_parts = 1 if self.gcn or self.pool else 2      # the GEMM parts that are rows of the source
        self.table = None

    def dense(self, x):
        """The [N+1, w] gradient of the rows this layer outputs: x itself, or the scatter of x into rows' ids."""
        if self.rows is None:
            return x
        return ops.embedding_grad([(self.rows, x.contiguous(), 1, 1.0)], self.graph.n_rows, x.shape[1])

    def table_grad(self, d):
        """The gradient of the layer's source table from d, the source gradient in the graph's row space."""
        if self.src_ids is None:
            return d
        return ops.embedding_grad([(self.src_ids, d, 1, 1.0)], self.table.shape[0], d.shape[1])

    def forward(self, h, kept):
        """The GEMM parts of the layer.  kept: None for inference, else a list that receives what the backward reads
        besides the parts."""
        agg, g, rows = self.agg, self.graph, self.rows
        self.table = h if self.src_ids is not None else None
        indptr, indices, h_rows = self.table_csr if self.table_csr is not None else (g.indptr, g.indices, rows)
        s = self.sites
        # the means' masks: the table CSR is the global one (positions by node id), else the graph's own map
        tgraph = FullNeighborGraph(indptr, indices) if self.table_csr is not None else g
        drop = {} if s is None or self.pool else {"dropout": (s["neigh"], s["self"], tgraph.pos_map)}
        if self.gcn:
            m = ops.csr_aggregate(h, indptr, indices, "mean_self", rows=h_rows, **drop)
            return [(m, agg.neigh_input_dim, agg.vars["weights"])]
        widen = h.dtype != torch.float32
        n = h.shape[0] if h_rows is None else h_rows.numel()
        hs = _rows(h, h_rows, 0, n, widen) if (widen or h_rows is not None) else h
        if not self.pool:
            if s is not None:                                        # the self rows by node id, after widening
                hs = ops.dropout_apply(hs, s["self"], pos_ids=tgraph.node_ids(h_rows), out=None if hs is h else hs)
            m = ops.csr_aggregate(h, indptr, indices, "mean", rows=h_rows, **drop)
            return [(hs, agg.input_dim, agg.vars["self_weights"]), (m, agg.neigh_input_dim, agg.vars["neigh_weights"])]
        if self.src_ids is None:
            x = z = _rows(h, None, 0, h.shape[0], True) if widen else h
        elif widen or s is not None:
            x = z = ops.gather_rows_f32(h, self.src_ids)             # V_0's rows, widened
        else:                                                        # V_0's rows read by id: no gathered copy
            x, z = None, ops.TableRows(h, [(self.src_ids, 0)], self.src_ids.numel())
        if s is not None:                                            # the MLP input, once per node, by node id
            x = z = ops.dropout_apply(x, s["mlp"], pos_ids=g.node_ids(None), out=None if x is h else x)
        for dense in agg.mlp_layers:                 # Dense without its dropout (layers.py:104-116), once per node
            code, post = act_code(dense.act)
            if getattr(dense, "_packed", None) is None:
                dense._packed = ops.PackedWeights()
            z = ops.sage_gemm([(z, dense.input_dim, dense.vars["weights"])], bias=dense.vars.get("bias"), act=code,
                              math=agg.math, packed=dense._packed)
            z = post(z) if post else z
        op = "max" if agg.pool == "max" else "mean"
        if kept is not None and op == "max" and rows is not None:
            # training: the backward needs every row's max - the same chains, then the rows
            p_all = ops.csr_aggregate(z, g.indptr, g.indices, "max")
            p = p_all.index_select(0, rows)
        else:
            p = p_all = ops.csr_aggregate(z, g.indptr, g.indices, op, rows=rows)
        if kept is not None:
            kept.extend([x, z, p_all])
        return [(hs, agg.input_dim, agg.vars["self_weights"]), (p, agg.hidden_dim, agg.vars["neigh_weights"])]

    def backward(self, xs, dxs, params, kept, cols):
        """(gradients of the pools' Wm, bm, d(source) [N + 1, cols] or None) from dxs, the gradients of the parts' rows."""
        for p in range(len(dxs)):                    # made dense in place: each row gradient is freed once scattered
            if dxs[p] is not None:
                dxs[p] = self.dense(dxs[p])
        s, g = self.sites, self.graph
        if self.gcn:
            return [], (g.mean_backward(dxs[0], True, s and (s["neigh"], s["self"])) if cols else None)
        dself = dxs[0]
        if not self.pool:
            if not cols:
                return [], None
            if s is not None:
                dself = ops.dropout_apply(dself, s["self"], pos_ids=g.node_ids(None), out=dself)
            return [], g.mean_backward(dxs[1], False, s and (s["neigh"], s["self"])) + dself
        (Wm, _), (x, z, p_all), dp = params, kept, dxs[1]
        if x is None:                                # the MLP read V_0's rows by id: gather them for dWm
            x = ops.gather_rows_f32(self.table, self.src_ids)
        if self.agg.pool == "max":
            t_indptr, t_indices = self.graph.transpose(False)
            dzp = ops.csr_max_backward(z, p_all, dp, self.graph.indptr, self.graph.indices, t_indptr, t_indices)
        else:
            dzp = self.graph.mean_backward(dp, False) * (z > 0).to(dp.dtype)    # the ReLU of the Dense layer
        K = Wm.shape[0]
        grads = [x[:, :K].t() @ dzp, dzp.sum(dim=0)]
        if not cols:
            return grads, None
        dx = dzp @ Wm[:cols].t()
        if s is not None:                                            # through the MLP input's node mask
            dx = ops.dropout_apply(dx, s["mlp"], pos_ids=g.node_ids(None), out=dx)
        return grads, dx + dself

    def source_grads(self, ctx, dsrc, dy):
        """(d(h) of a layer >= 1, d(embeddings) of layer 0 with identity_dim > 0) from the source gradient dsrc."""
        demb = self.table_grad(dsrc[:, :ctx.emb_shape[1]]) if ctx.emb_shape is not None and dsrc is not None else None
        return (dsrc if ctx.src_needs_grad else None), demb


class _L2NormalizeFn(torch.autograd.Function):
    """tf.nn.l2_normalize(x, 1) through gs_l2_normalize_rows (the bits of full_neighbor_embeddings); the backward is the
    formula's gradient."""

    @staticmethod
    def forward(ctx, x):
        ctx.save_for_backward(x)
        return ops.l2_normalize_rows_(x.detach().contiguous().clone())

    @staticmethod
    def backward(ctx, dy):
        (x,) = ctx.saved_tensors
        with torch.enable_grad():
            xx = x.detach().requires_grad_(True)
            out = xx / torch.sqrt(torch.clamp((xx * xx).sum(dim=1, keepdim=True), min=1e-12))
            return torch.autograd.grad(out, xx, dy)[0]


def refuse_capture(what):
    if torch.cuda.is_available() and torch.cuda.is_current_stream_capturing():
        raise NotImplementedError("%s cannot be captured in a CUDA graph" % what)


def refuse_full_neighbor(model, training, dropout=None):
    """The NotImplementedErrors of the full-neighbourhood entry points; training adds those of the training paths.
    dropout: the training call's explicit rate (None: the model's dropout_rate must be 0)."""
    what = "training" if training else "inference"
    if model.aggregator_cls is SeqAggregator:
        raise NotImplementedError("full-neighbourhood %s is not implemented for the seq aggregator (its neighbour "
                                  "order is the sampled order)" % what)
    if hasattr(model.features, "c_table"):
        raise NotImplementedError("full-neighbourhood %s with a node-partitioned (ShardedFeatures) table is not "
                                  "implemented" % what)
    refuse_host_table(model.features, "full-neighbourhood %s (it reads the whole table)" % what)
    refuse_int8_table(model.features, "full-neighbourhood %s" % what)
    if not training:
        return
    if model.aggregator_cls is TwoMaxLayerPoolingAggregator:
        raise NotImplementedError("full-neighbourhood training is not implemented for the twomaxpool aggregator (the "
                                  "backward through its second Dense layer has no full-neighbourhood form)")
    if getattr(model, "distributed", False):
        raise NotImplementedError("full-neighbourhood training with distributed=True is not implemented")
    if dropout is None and getattr(model, "dropout_rate", 0.):
        raise NotImplementedError("full-neighbourhood training with dropout > 0 is not implemented (the masks are "
                                  "defined per sampled copy of a row; a whole neighbourhood has no such copies) - pass "
                                  "dropout=model.dropout_rate for the full-neighbourhood masks, one per CSR entry and "
                                  "per node")
    refuse_capture("a full-neighbourhood training step")


def full_neighbor_graph(model, indptr, indices):
    """The model's cached FullNeighborGraph for this CSR (rebuilt when the CSR tensors change)."""
    g = getattr(model, "_full_neighbor_graph", None)
    if g is None or g.key != FullNeighborGraph.key_of(indptr, indices):
        g = model._full_neighbor_graph = FullNeighborGraph(indptr, indices)
    return g


def _inputs(model, indptr, indices, node_ids):
    """(indptr, indices, ids): the CSR on the model's device, checked, and node_ids (None: all N nodes) as int32 with
    every id outside [0, N) named N - it reads the dummy node in the forward; naming it N routes its gradient there too
    (same bits)."""
    n_rows = int(model.features.shape[0])
    indptr, indices = model._csr_input(indptr, torch.int64, "indptr"), model._csr_input(indices, torch.int32, "indices")
    if indptr.dim() != 1 or indptr.numel() != n_rows:
        raise ValueError("indptr must have N + 1 = %d entries (one row per node of the [N+1, .] table, plus the end)"
                         % n_rows)
    if node_ids is None:
        return indptr, indices, torch.arange(n_rows - 1, dtype=torch.int32, device=model.device)
    ids = torch.as_tensor(node_ids).to(device=model.device, dtype=torch.int32).reshape(-1)
    ids = torch.where((ids < 0) | (ids >= n_rows - 1), torch.full_like(ids, n_rows - 1), ids)
    return indptr, indices, ids


def minibatch_layers(aggregators, indptr, indices, ids):
    """One _FullLayer per aggregator over the blocks of ops.csr_blocks(indptr, indices, ids, L) (ids clamped)."""
    L = len(aggregators)
    blocks = ops.csr_blocks(indptr, indices, ids, L)
    layers = []
    for layer, (agg, b) in enumerate(zip(aggregators, blocks)):
        graph = FullNeighborGraph(b.indptr, b.indices, pos_map=(indptr, b.src_ids, indices.numel()))
        if layer == 0:
            v1 = blocks[1].src_ids if L > 1 else ids
            layers.append(_FullLayer(agg, graph, b.rows, src_ids=b.src_ids, table_csr=(indptr, indices, v1)))
        else:
            layers.append(_FullLayer(agg, graph, b.rows))
    return layers


def _layers(model, indptr, indices, node_ids, training, minibatch, dropout=None):
    """The checked layers of one call: over the receptive-field blocks of node_ids (minibatch; reads the block sizes
    back once), else over the whole CSR - the model's cached FullNeighborGraph when training, an uncached one otherwise
    (inference builds no transposes, and must not evict the ones a training CSR has cached)."""
    refuse_full_neighbor(model, training, dropout)
    if minibatch:
        refuse_capture("a full-neighbourhood minibatch (it reads the block sizes back)")
    indptr, indices, ids = _inputs(model, indptr, indices, node_ids)
    if model.aggregators is None:
        model.aggregators = build_aggregators(model)
    if minibatch:
        return minibatch_layers(model.aggregators, indptr, indices, ids)
    graph = full_neighbor_graph(model, indptr, indices) if training else FullNeighborGraph(indptr, indices)
    L = len(model.aggregators)
    return [_FullLayer(agg, graph, ids if layer == L - 1 else None) for layer, agg in enumerate(model.aggregators)]


def full_neighbor_embeddings(model, indptr, indices, node_ids=None, normalize=True, minibatch=False):
    """SampleAndAggregate.full_neighbor_embeddings (minibatch: full_neighbor_minibatch_embeddings), without autograd."""
    h = model.features
    with torch.no_grad():
        for fl in _layers(model, indptr, indices, node_ids, False, minibatch):
            h = fl.agg._finish(fl.forward(h, None), fl.agg._combine())
        if normalize:
            h = ops.l2_normalize_rows_(h.contiguous())
    return h


def full_neighbor_outputs(model, indptr, indices, node_ids, normalize=True, minibatch=False, dropout=None):
    """full_neighbor_embeddings(indptr, indices, node_ids, normalize, minibatch) with an autograd graph over the
    aggregator weights and (identity_dim > 0) model.embeds.  Same values, bit for bit.  dropout = p > 0: the layers'
    sites of full_neighbor_site_plan, numbered from model.dropout_counter, which advances past them."""
    p = check_full_neighbor_dropout(dropout)
    layers = _layers(model, indptr, indices, node_ids, True, minibatch, dropout=p)
    if p:
        pool = isinstance(layers[0].agg, MaxPoolingAggregator)
        plan = full_neighbor_site_plan("maxpool" if pool else "mean", len(layers))
        for i, (layer, role) in enumerate(plan):
            layers[layer].sites = layers[layer].sites or {}
            layers[layer].sites[role] = (model.dropout_key, model.dropout_counter + i, p)
        model.dropout_counter += len(plan)
    h = model.features
    for layer, fl in enumerate(layers):
        emb = getattr(model, "embeds", None) if layer == 0 else None
        h = _LayerFn.apply(fl, h, emb, *layer_params(fl.agg))
    return _L2NormalizeFn.apply(h) if normalize else h
