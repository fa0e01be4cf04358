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

Sampled minibatches (sampled_minibatch_*; contract: oracle/sampled_blocks.py) run the same layers over blocks whose rows
keep at most k_l sampled entries (ops.csr_blocks with fanouts).  Layer 0 cannot reduce the global table through the
global CSR, since its rows are sampled: the means reduce block 0 over V_0's rows (gathered by id, widened to fp32), the
pools' MLP reads V_0's rows by id as before; the self rows are V_1's table rows by id in both.  Everything else is the
minibatch path.  The draws are keyed by the model's neigh_sampler (seed, counter); one block set advances the counter by 1.
Over a host (HostFeatures) or int8 (Int8Features) table, layer 0 runs in block-local space instead, as every layer >= 1
does: X0 = V_0's rows as fp32 (HostFeatures.gather_rows_f32: cache or host link in one pass; ops.gather_rows_f32 for a
device int8 table), then _FullLayer(agg, block 0, block 0's rows = V_1's positions in V_0) over X0.  Its operands are the
fp32 values the device table's layer 0 reads, in the same order and layout, so the bits are the same; only V_0 is read.

Training dropout (dropout=p > 0; contract: oracle/full_neighbor_dropout.py) masks by global identities: per CSR entry for
the means' neighbour branch (gs_csr_aggregate_dropout, the entry's global CSR position), per node for the mean's self
rows, GCN's own row and the pools' MLP input (ops.dropout_apply by id).  Each graph carries the position map of its
kernels - (indptr, None, nnz) for the whole graph, (global indptr, src_ids, global nnz) for a block - so a block masks every
element as the whole-graph pass does.  The backward regenerates every mask: the transposed sum reads the transpose's
t_slot (ops.csr_transpose(slots=True)) to find each entry's forward position.  A sampled block (contract:
oracle/sampled_blocks_dropout.py) keeps only some entries of each raw row, so its map carries a fourth element, each
entry's offset in its raw row (ops.csr_blocks(..., entry_offsets=True)): the forward masks entry j at pos_indptr[g] +
offset, and the backward maps t_slot through the offsets (ops.csr_slots_to_offsets) before the same transposed sum.  A
sampled entry is then masked as the same edge is in the whole-graph pass.

Edge weights (edge_weight=w, fp32, one per CSR entry; contract: oracle/weighted.py) scale each message before the
reduction: every reduction runs gs_csr_aggregate_weighted with its graph's per-entry weights, the means' backward sums
fl(w * g / count) over the transpose with each transposed entry's forward weight (ops.csr_transpose_weights, cached on
the FullNeighborGraph beside the transposes), and the max-pool backward splits ties on the weighted values
(ops.csr_max_backward with weights).  A block's entries carry the weights of the raw entries they copy
(ops.csr_block_weights, built per call); layer 0 of a whole-neighbourhood minibatch reads the global CSR, so it takes w.
Not with training dropout p > 0.

Weighted draws (sample_weight=w, fp32, one per CSR entry; contract: oracle/weighted_sampling.py) change only how the
sampled blocks choose their entries: ops.csr_blocks(..., sample_weights=w) keeps at most k_l of each row's entries with
w > 0, drawn in proportion to w.  The blocks have the uniform blocks' layout and offsets, so every layer, mask, edge
weight and table above runs on them unchanged.
"""
import numpy as np
import torch

from . import ops
from .aggregators import GCNAggregator, MaxPoolingAggregator, SeqAggregator, TwoMaxLayerPoolingAggregator, _rows
from .host_features import HostFeatures, refuse_host_table
from .int8_features import is_int8_table, refuse_int8_table
from .layers import act_code
from .supervised_models import (_LayerFn, build_aggregators, check_full_neighbor_dropout, full_neighbor_site_plan,
                                layer_params, refuse_dropout_table)


class FullNeighborGraph(object):
    """The transposes and divisors of one CSR, built on first use.  `key` identifies the CSR tensors (data_ptr, numel,
    _version of both); the tensors themselves are held, so their memory cannot be reused by a different CSR while cached."""

    def __init__(self, indptr, indices, pos_map=None, weights=None):
        """pos_map: (pos_indptr, pos_ids or None, pos_nnz[, pos_off]), how the masks name this CSR's rows and entries
        globally (default: the CSR is the global one); pos_off: a sampled block's per-entry raw-row offsets.  weights:
        None, or fp32 [len(indices)], the edge weights of this CSR's entries (part of the key)."""
        self.indptr, self.indices, self.weights = indptr, indices, weights
        self.pos_map = pos_map if pos_map is not None else (indptr, None, indices.numel())
        self.key = FullNeighborGraph.key_of(indptr, indices, weights)
        self.n_rows = indptr.numel()                 # N + 1
        self._t, self._counts, self._tw = {}, {}, {}

    @staticmethod
    def key_of(indptr, indices, weights=None):
        ts = (indptr, indices) if weights is None else (indptr, indices, weights)
        return tuple((t.data_ptr(), t.numel(), t._version) for t in ts)

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

    def t_weights(self, with_self):
        """The edge weights of transpose(with_self)'s entries, aligned with its t_indices (ops.csr_transpose_weights)."""
        if with_self not in self._tw:
            _, t_indices, t_slot = self.transpose(with_self, slots=True)
            self._tw[with_self] = ops.csr_transpose_weights(self.weights, self.indptr, t_indices, t_slot)
        return self._tw[with_self]

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
        if self.weights is not None:                 # no dropout with weights
            t_indptr, t_indices = self.transpose(with_self, slots=True)[:2]
            return ops.csr_aggregate(gp, t_indptr, t_indices, "sum", weights=self.t_weights(with_self))
        if sites is None:
            t_indptr, t_indices = self.transpose(with_self)
            return ops.csr_aggregate(gp, t_indptr, t_indices, "sum")
        t_indptr, t_indices, t_slot = self.transpose(with_self, slots=True)
        if len(self.pos_map) == 4:                   # a sampled block: slots in the block row -> offsets in the raw row
            t_slot = ops.csr_slots_to_offsets(t_slot, t_indices, self.indptr, self.pos_map[3])
        return ops.csr_aggregate(gp, t_indptr, t_indices, "sum", dropout=(sites[0], sites[1], self.pos_map[:3]),
                                 t_slot=t_slot)

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

    def __init__(self, agg, graph, rows, src_ids=None, table_csr=None, self_ids=None, x0_dtype=None):
        """table_csr: (global indptr, global indices, V_1's global ids, global edge weights or None).
        self_ids (a sampled block 0, with src_ids and no table_csr): V_1's global ids - the self rows are read from the
        table by id, and the reductions run over the block itself, the means' on V_0's gathered rows.
        x0_dtype (a sampled block 0 in block-local space, no src_ids): the source is X0, V_0's rows of a table of this
        dtype read as fp32 for this call only - the self rows are laid out as that table's own layer 0 lays them out
        (widened rows padded), and X0 may be masked in place."""
        self.agg, self.graph, self.rows = agg, graph, rows
        self.src_ids, self.table_csr, self.self_ids, self.x0_dtype = src_ids, table_csr, self_ids, x0_dtype
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
        indptr, indices, h_rows, w = self.table_csr if self.table_csr is not None else (g.indptr, g.indices, rows,
                                                                                        g.weights)
        hn, n_rows = h, h_rows                  # the means' reduction source and its rows
        if self.self_ids is not None:           # a sampled block 0: self rows by global id, reductions in the block
            h_rows = self.self_ids
            if not self.pool:
                hn = ops.gather_rows_f32(h, self.src_ids)
        s = self.sites
        # the means' masks: the table CSR is the global one (positions by node id), else the graph's own map
        tgraph = FullNeighborGraph(indptr, indices) if self.table_csr is not None else g
        drop = {} if s is None or self.pool else {"dropout": (s["neigh"], s["self"], tgraph.pos_map)}
        if w is not None:                            # the edge weights of the means' CSR (no dropout with them)
            drop = {"weights": w}
        if self.gcn:
            m = ops.csr_aggregate(hn, indptr, indices, "mean_self", rows=n_rows, **drop)
            return [(m, agg.neigh_input_dim, agg.vars["weights"])]
        widen = h.dtype != torch.float32
        n = h.shape[0] if h_rows is None else h_rows.numel()
        wself = widen if self.x0_dtype is None else self.x0_dtype != torch.float32
        hs = _rows(h, h_rows, 0, n, wself) if (wself or h_rows is not None) else h
        if not self.pool:
            if s is not None:                                        # the self rows by node id, after widening
                # a sampled block 0 reads them by global id (self_ids), which are their positions
                ids = h_rows if self.self_ids is not None else tgraph.node_ids(h_rows)
                hs = ops.dropout_apply(hs, s["self"], pos_ids=ids, out=None if hs is h else hs)
            m = ops.csr_aggregate(hn, indptr, indices, "mean", rows=n_rows, **drop)
            return [(hs, agg.input_dim, agg.vars["self_weights"]), (m, agg.neigh_input_dim, agg.vars["neigh_weights"])]
        if self.src_ids is None:
            x = z = _rows(h, None, 0, h.shape[0], True) if widen else h
        elif widen or s is not None:
            x = z = ops.gather_rows_f32(h, self.src_ids)             # V_0's rows, widened
        else:                                                        # V_0's rows read by id: no gathered copy
            x, z = None, ops.TableRows(h, [(self.src_ids, 0)], self.src_ids.numel())
        if s is not None:                                            # the MLP input, once per node, by node id
            # X0 is this call's own buffer: masked in place, as the table path masks its gathered copy
            own = x is not h or self.x0_dtype is not None
            x = z = ops.dropout_apply(x, s["mlp"], pos_ids=g.node_ids(None), out=x if own else None)
        for dense in agg.mlp_layers:                 # Dense without its dropout (layers.py:104-116), once per node
            code, post = act_code(dense.act)
            if getattr(dense, "_packed", None) is None:
                dense._packed = ops.PackedWeights()
            z = ops.sage_gemm([(z, dense.input_dim, dense.vars["weights"])], bias=dense.vars.get("bias"), act=code,
                              math=agg.math, packed=dense._packed)
            z = post(z) if post else z
        op = "max" if agg.pool == "max" else "mean"
        gw = {} if g.weights is None else {"weights": g.weights}
        if kept is not None and op == "max" and rows is not None:
            # training: the backward needs every row's max - the same chains, then the rows
            p_all = ops.csr_aggregate(z, g.indptr, g.indices, "max", **gw)
            p = p_all.index_select(0, rows)
        else:
            p = p_all = ops.csr_aggregate(z, g.indptr, g.indices, op, rows=rows, **gw)
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
        if self.agg.pool == "max" and g.weights is not None:
            t_indptr, t_indices = g.transpose(False, slots=True)[:2]
            dzp = ops.csr_max_backward(z, p_all, dp, g.indptr, g.indices, t_indptr, t_indices, weights=g.weights,
                                       t_weights=g.t_weights(False))
        elif self.agg.pool == "max":
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


def refuse_full_neighbor(model, training, dropout=None, tables=True):
    """The NotImplementedErrors of the full-neighbourhood entry points; training adds those of the training paths.
    dropout: the training call's explicit rate (None: the model's dropout_rate must be 0).  tables=False leaves out the
    host- and int8-table refusals (the sampled blocks read V_0's rows only)."""
    what = "training" if training else "inference"
    if model.aggregator_cls is SeqAggregator:
        raise NotImplementedError("full-neighbourhood %s is not implemented for the seq aggregator (its neighbour "
                                  "order is the sampled order)" % what)
    if hasattr(model.features, "c_table"):
        raise NotImplementedError("full-neighbourhood %s with a node-partitioned (ShardedFeatures) table is not "
                                  "implemented" % what)
    if tables:
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


def full_neighbor_graph(model, indptr, indices, weights=None):
    """The model's cached FullNeighborGraph for this CSR and edge weights (rebuilt when the tensors change)."""
    g = getattr(model, "_full_neighbor_graph", None)
    if g is None or g.key != FullNeighborGraph.key_of(indptr, indices, weights):
        g = model._full_neighbor_graph = FullNeighborGraph(indptr, indices, weights=weights)
    return g


def refuse_weighted_dropout(edge_weight, dropout):
    """edge_weight together with training dropout p > 0 is not implemented."""
    if edge_weight is not None and dropout:
        raise NotImplementedError("edge_weight with training dropout > 0 is not implemented (pass dropout=None or 0, "
                                  "or no edge_weight)")


def edge_weights(model, edge_weight, indices, name="edge_weight"):
    """edge_weight as a 1-D fp32 tensor on the model's device, one weight per entry of indices: numpy arrays are
    uploaded, tensors must already be there (TypeError: not float32; ValueError: wrong length or device).  No check of
    the values: that would synchronise with the host.  name: the keyword the errors name (sample_weight too)."""
    if edge_weight is None:
        return None
    if not torch.is_tensor(edge_weight):
        arr = np.asarray(edge_weight)
        if arr.dtype != np.float32:
            raise TypeError("%s must be float32 (got %s)" % (name, arr.dtype))
        edge_weight = torch.as_tensor(arr, device=model.device)
    if edge_weight.dtype != torch.float32:
        raise TypeError("%s must be float32 (got %s)" % (name, edge_weight.dtype))
    if edge_weight.device != indices.device:
        raise ValueError("%s must be on the model's device %s (got %s)" % (name, indices.device, edge_weight.device))
    if edge_weight.dim() != 1 or edge_weight.numel() != indices.numel():
        raise ValueError("%s needs one weight per CSR entry: shape (%d,), got %s"
                         % (name, indices.numel(), tuple(edge_weight.shape)))
    return edge_weight.contiguous()


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


def minibatch_layers(aggregators, indptr, indices, ids, draw=None, dropout=0., x0_dtype=None, weights=None):
    """One _FullLayer per aggregator over the blocks of ops.csr_blocks(indptr, indices, ids, L) (ids clamped); draw =
    (fanouts, seed, call[, sample weights]): over the sampled blocks of ops.csr_blocks(..., fanouts, seed, call,
    sample_weights=) instead (a None or absent fourth element: uniform draws), and with
    dropout = p > 0 each block's position map also carries its entries' raw-row offsets.  x0_dtype (sampled): layer 0
    runs in block-local space over X0, V_0's fp32 rows of a table of that dtype (sampled_layer0_rows).  weights: the
    global edge weights; each block then carries those of the raw entries it copies (ops.csr_block_weights)."""
    L = len(aggregators)
    offsets = [None] * L
    if draw is None:
        blocks = ops.csr_blocks(indptr, indices, ids, L)
    else:
        fanouts, seed, call = draw[:3]
        sw = {} if len(draw) < 4 or draw[3] is None else {"sample_weights": draw[3]}
        if dropout or weights is not None:
            blocks, offsets = ops.csr_blocks(indptr, indices, ids, L, fanouts=fanouts, seed=seed, call=call,
                                             entry_offsets=True, **sw)
        else:
            blocks = ops.csr_blocks(indptr, indices, ids, L, fanouts=fanouts, seed=seed, call=call, **sw)
    layers = []
    for layer, (agg, b) in enumerate(zip(aggregators, blocks)):
        pos_map = (indptr, b.src_ids, indices.numel()) + ((offsets[layer],) if offsets[layer] is not None else ())
        bw = None if weights is None else ops.csr_block_weights(weights, indptr, b, offsets[layer])
        graph = FullNeighborGraph(b.indptr, b.indices, pos_map=pos_map, weights=bw)
        if layer == 0:
            v1 = blocks[1].src_ids if L > 1 else ids
            if draw is not None and x0_dtype is not None:
                layers.append(_FullLayer(agg, graph, b.rows, x0_dtype=x0_dtype))
            elif draw is not None:
                layers.append(_FullLayer(agg, graph, b.rows, src_ids=b.src_ids, self_ids=v1))
            else:
                layers.append(_FullLayer(agg, graph, b.rows, src_ids=b.src_ids,
                                         table_csr=(indptr, indices, v1, weights)))
        else:
            layers.append(_FullLayer(agg, graph, b.rows))
    return layers


def refuse_sampled(model, training, dropout=None):
    """The NotImplementedErrors of the sampled-block entry points: refuse_full_neighbor's but its host- and int8-table
    ones, CUDA-graph capture and, when training, dropout=None on a model with dropout_rate > 0 and dropout = p > 0 on an
    int8 table."""
    if training and dropout is None and getattr(model, "dropout_rate", 0.):
        raise NotImplementedError("sampled-block training with dropout > 0 needs the rate passed explicitly - pass "
                                  "dropout=model.dropout_rate for the per-edge masks keyed by global CSR positions "
                                  "(oracle/sampled_blocks_dropout.py)")
    refuse_full_neighbor(model, training, dropout, tables=False)
    if training and dropout and is_int8_table(model.features):
        refuse_dropout_table(model.features)
    refuse_capture("a sampled-block minibatch (it reads the block sizes back)")


def reads_v0_rows(features):
    """Whether a sampled block set's layer 0 runs over X0, V_0's rows as fp32: a host table (only V_0 crosses the link)
    or an int8 table (V_0 dequantised once).  fp32 and bf16 device tables are read by id in place."""
    return isinstance(features, HostFeatures) or is_int8_table(features)


def sampled_layer0_rows(features, src_ids):
    """X0: the rows src_ids (V_0) of a host or int8 table as an fp32 [|V_0|, pad_cols(F)] buffer's [:, :F] view, the
    layout ops.gather_rows_f32 gives - HostFeatures.gather_rows_f32 for a host table, ops.gather_rows_f32 for a device
    int8 one."""
    if isinstance(features, HostFeatures):
        return features.gather_rows_f32(src_ids)
    return ops.gather_rows_f32(features, src_ids)


def sampled_draw(model):
    """(fanouts, seed, call) of one sampled block set - block l takes layer_infos[l].num_samples, the draws are keyed by
    the neigh_sampler's seed at its counter - and advances that counter by 1."""
    sampler = model.layer_infos[0].neigh_sampler
    fanouts = ops.check_fanouts([info.num_samples for info in model.layer_infos], len(model.layer_infos))
    call = int(sampler.counter)
    sampler.counter = call + 1
    return fanouts, int(sampler.seed), call


def _layers(model, indptr, indices, node_ids, training, minibatch, dropout=None, sampled=False, edge_weight=None,
            sample_weight=None):
    """(the checked layers of one call, layer 0's source): over the receptive-field blocks of node_ids (minibatch; reads
    the block sizes back once; sampled: over sampled blocks), else over the whole CSR - the model's cached
    FullNeighborGraph when training, an uncached one otherwise (inference builds no transposes, and must not evict the
    ones a training CSR has cached).  The source is the model's table, or X0 for sampled blocks over a host or int8
    table.  edge_weight: None, or one fp32 weight per CSR entry (edge_weights).  sample_weight (sampled only): None, or
    one fp32 weight per CSR entry that the sampled blocks draw in proportion to."""
    if sampled:
        refuse_sampled(model, training, dropout)
    else:
        refuse_full_neighbor(model, training, dropout)
    refuse_weighted_dropout(edge_weight, dropout)
    if minibatch:
        refuse_capture("a full-neighbourhood minibatch (it reads the block sizes back)")
    indptr, indices, ids = _inputs(model, indptr, indices, node_ids)
    w = edge_weights(model, edge_weight, indices)
    sw = edge_weights(model, sample_weight, indices, "sample_weight")
    if model.aggregators is None:
        model.aggregators = build_aggregators(model)
    h = model.features
    if sampled:
        x0 = reads_v0_rows(h)
        layers = minibatch_layers(model.aggregators, indptr, indices, ids, draw=sampled_draw(model) + (sw,),
                                  dropout=dropout, x0_dtype=h.dtype if x0 else None, weights=w)
        # |V_0| is known from the block build's size read: X0 is sized without another
        return layers, (sampled_layer0_rows(h, layers[0].graph.pos_map[1]) if x0 else h)
    if minibatch:
        return minibatch_layers(model.aggregators, indptr, indices, ids, weights=w), h
    graph = (full_neighbor_graph(model, indptr, indices, w) if training else
             FullNeighborGraph(indptr, indices, weights=w))
    L = len(model.aggregators)
    return [_FullLayer(agg, graph, ids if layer == L - 1 else None) for layer, agg in enumerate(model.aggregators)], h


def full_neighbor_embeddings(model, indptr, indices, node_ids=None, normalize=True, minibatch=False, sampled=False,
                             edge_weight=None, sample_weight=None):
    """SampleAndAggregate.full_neighbor_embeddings (minibatch: full_neighbor_minibatch_embeddings; sampled:
    sampled_minibatch_embeddings), without autograd."""
    with torch.no_grad():
        layers, h = _layers(model, indptr, indices, node_ids, False, minibatch, sampled=sampled, edge_weight=edge_weight,
                            sample_weight=sample_weight)
        for fl in layers:
            h = fl.agg._finish(fl.forward(h, None), fl.agg._combine())
        if normalize:
            h = ops.l2_normalize_rows_(h.contiguous())
    return h


def full_neighbor_outputs(model, indptr, indices, node_ids, normalize=True, minibatch=False, dropout=None,
                          sampled=False, edge_weight=None, sample_weight=None):
    """full_neighbor_embeddings(indptr, indices, node_ids, normalize, minibatch, sampled) with an autograd graph over the
    aggregator weights and (identity_dim > 0) model.embeds.  Same values, bit for bit.  dropout = p > 0: the layers'
    sites of full_neighbor_site_plan, numbered from model.dropout_counter, which advances past them.  edge_weight: the
    CSR's per-entry weights (oracle/weighted.py).  sample_weight (sampled): the weights the blocks draw by
    (oracle/weighted_sampling.py)."""
    p = check_full_neighbor_dropout(dropout)
    layers, h = _layers(model, indptr, indices, node_ids, True, minibatch, dropout=p, sampled=sampled,
                        edge_weight=edge_weight, sample_weight=sample_weight)
    if p:
        pool = isinstance(layers[0].agg, MaxPoolingAggregator)
        plan = full_neighbor_site_plan("maxpool" if pool else "mean", len(layers))
        for i, (layer, role) in enumerate(plan):
            layers[layer].sites = layers[layer].sites or {}
            layers[layer].sites[role] = (model.dropout_key, model.dropout_counter + i, p)
        model.dropout_counter += len(plan)
    for layer, fl in enumerate(layers):
        emb = getattr(model, "embeds", None) if layer == 0 else None
        h = _LayerFn.apply(fl, h, emb, *layer_params(fl.agg))
    return _L2NormalizeFn.apply(h) if normalize else h
