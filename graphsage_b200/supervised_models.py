"""SupervisedGraphsage - the training step around the hot path (SURVEY section 8f row 1; reference
graphsage/supervised_models.py:10-126).

Forward: the library's CUDA kernels (sample -> fused gather+mean -> wgmma / fp32 GEMM), wrapped in
torch.autograd.Function so the step is differentiable.  Backward: the gradient formulas of the mean / GCN
aggregators, with the weight-gradient GEMMs (X^T dZ) as plain library matmuls (torch / cuBLAS fp32).  Features are
not trainable; with identity_dim > 0 the embedding columns of the layer-0 table are, and their gradient is scattered
into a dense [N+1, d] table by the library's deterministic embedding-gradient kernel (ops.embedding_grad).  Head
(l2_normalize -> Dense -> sigmoid / softmax cross-entropy + weight decay), gradient clipping to +-5 and Adam follow
supervised_models.py:85-126.

Training dropout (placeholders['dropout'] = p > 0; reference aggregators.py:46-47 / 104-105, layers.py:107,
supervised_models.py:88-90) follows the Philox mask contract of include/graphsage_b200.h (gs_dropout_site): the forward
drops the gathered rows inside the fused gather (mean / GCN) or the pools' MLP input and the head input, and the backward
regenerates the same masks instead of storing them.  A pass numbers its sites in the reference's call order
(dropout_site_plan); the model's host `dropout_counter` gives the first call number and advances past them.
"""
import torch

from . import ops
from .graphed_training import GraphedTrainStep
from .host_features import refuse_host_table, stage_layer0
from .int8_features import refuse_int8_table
from .layers import act_code, identity, relu  # noqa: F401
from .aggregators import (FUSED_POOL_HIDDEN_STEP, FUSED_POOL_MAX_FANOUT, FUSED_POOL_MAX_K, TwoMaxLayerPoolingAggregator,
                          fused_pool_fits)
from .models import _SIZED_AGGREGATORS, SampleAndAggregate, layer_segments


def _embedding_grad(emb_shape, lists, sites=None):
    """The layer-0 gradient w.r.t. the embedding columns [0, d) of the table: (ids, grad rows, group, scale) lists, and with
    dropout one (seed, call, rate) site per list."""
    return ops.embedding_grad(lists, emb_shape[0], emb_shape[1], sites=sites)


def dropout_site_plan(kind, n_layers, head=False):
    """The dropout sites of one forward pass in the reference's call order (models.py:303-328 calls each layer's
    aggregator once per hop): [(layer, hop, role)], role "neigh" then "self" for mean / gcn (aggregators.py:46-47,
    104-105), the one "mlp" input of the pools' Dense (layers.py:107), then (None, None, "head") for the supervised head
    (supervised_models.py:88-90); "seq" has no aggregator sites.  Site i of a pass draws with call = first call + i."""
    plan = []
    if kind == "seq":                   # SeqAggregator._call applies no dropout (aggregators.py:405-449): the head only
        n_layers = 0
    roles = {"maxpool": ("mlp",), "meanpool": ("mlp",), "twomaxpool": ("mlp", "mlp2")}.get(kind, ("neigh", "self"))
    for layer in range(n_layers):
        for hop in range(n_layers - layer):
            plan += [(layer, hop, role) for role in roles]
    return plan + ([(None, None, "head")] if head else [])


def full_neighbor_site_plan(kind, n_layers, head=False):
    """The dropout sites of one full-neighbourhood training pass (contract: oracle/full_neighbor_dropout.py): [(layer,
    role)], per layer "neigh" then "self" for mean / gcn - one mask per CSR entry, one per node - or the one per-node
    "mlp" input of the pools (the full path runs the MLP once per node), then (None, "head") for the supervised head.  Site
    i draws with call = first call + i."""
    roles = ("mlp",) if kind in ("maxpool", "meanpool") else ("neigh", "self")
    return [(layer, role) for layer in range(n_layers) for role in roles] + ([(None, "head")] if head else [])


def check_full_neighbor_dropout(dropout):
    """The `dropout` argument of the full_neighbor_* training methods: None (no masks; a model whose dropout_rate > 0 is
    refused), or a rate p in [0, 1) applied as asked - p = 0 draws nothing.  Anything else is a ValueError."""
    if dropout is None:
        return None
    if isinstance(dropout, bool) or not isinstance(dropout, (int, float)) or not 0.0 <= float(dropout) < 1.0:
        raise ValueError("dropout must be None or a rate in [0, 1) (got %r)" % (dropout,))
    return float(dropout)


class _DropoutFn(torch.autograd.Function):
    """y = drop(x) for one site (the supervised head's input, layers.py:107); the backward applies the same mask."""

    @staticmethod
    def forward(ctx, x, site):
        ctx.site = site
        return ops.dropout_apply(x.detach(), site)

    @staticmethod
    def backward(ctx, dy):
        return ops.dropout_apply(dy.contiguous(), ctx.site), None


def pool_branch_backward(pool, xn, h, hp, dhp, Wm, k, need_dx):
    """Gradients through hp = pool_k(h), h = relu(xn @ Wm + bm) for one hop (reference aggregators.py:176-182 /
    :256-262 backwards).  xn [n*k, F], h [n*k, hid] (post-ReLU), hp / dhp [n, hid].
    max: the gradient of a maximum goes to the positions that attain it, split evenly among ties (TensorFlow's
    reduce_max gradient); mean: dhp / k to every position.  Returns (dWm, dbm, dxn or None)."""
    n, hid = hp.shape
    h3 = h.reshape(n, k, hid)
    if pool == "max":
        sel = h3 == hp.unsqueeze(1)
        share = dhp / sel.sum(dim=1).to(dhp.dtype)
        dh = sel.to(dhp.dtype) * share.unsqueeze(1)
    else:
        dh = (dhp / float(k)).unsqueeze(1).expand(n, k, hid)
    dpre = (dh * (h3 > 0).to(dhp.dtype)).reshape(n * k, hid)             # ReLU of the Dense layer
    dWm = xn.t() @ dpre
    dbm = dpre.sum(dim=0)
    return dWm, dbm, (dpre @ Wm.t() if need_dx else None)


class _LayerFn(torch.autograd.Function):
    """y = agg.aggregate_rows(src, segments) for one aggregator layer, differentiable w.r.t. the layer's parameters,
    (layers >= 1, where rows are addressed by ranges) src, and (layer 0, identity_dim > 0) `emb`, the [N+1, d] embedding
    view of src's first d columns.  The per-kind work is the branch's (_AggregateRowsFn, _PoolAggregateRowsFn,
    _FusedPoolAggregateRowsFn, _SeqAggregateRowsFn, whose apply is the layer's entry, and the whole-neighbourhood
    full_neighbor_training._FullLayer): its forward gives the GEMM parts y = act(concat_or_add(x_p @ W_p) + bias)
    combines, its backward turns the gradients of its parts' inputs into the gradients of its own parameters and the
    source gradient its source_grads routes (the sampled branches: per-segment contributions, _source_grads)."""

    @staticmethod
    def forward(ctx, branch, src, emb, *params):
        agg = branch.agg
        code, post = act_code(agg.act)
        if post is not None:
            raise NotImplementedError("training supports act=relu or identity")
        with torch.no_grad():
            kept = []
            parts = branch.forward(src, kept)
            y = agg._finish(parts, agg._combine())
        ctx.branch, ctx.relu, ctx.concat = branch, code == ops.ACT_RELU, bool(agg.concat)
        ctx.src_shape, ctx.F_in, ctx.Ks = tuple(src.shape), src.shape[1], [K for _, K, _ in parts]
        ctx.src_needs_grad = bool(torch.is_tensor(src) and src.requires_grad)
        ctx.emb_shape = tuple(emb.shape) if emb is not None and emb.requires_grad else None
        ctx.n_params = len(params)
        ctx.save_for_backward(*[x for x, _, _ in parts], y, *params, *kept)
        return y

    @staticmethod
    def backward(ctx, dy):
        P = len(ctx.Ks)
        saved = ctx.saved_tensors
        xs, y, params, kept = saved[:P], saved[P], saved[P + 1:P + 1 + ctx.n_params], saved[P + 1 + ctx.n_params:]
        dz = dy * (y > 0).to(dy.dtype) if ctx.relu else dy
        D = params[0].shape[1]
        dzs = (dz[:, :D], dz[:, D:]) if P == 2 and ctx.concat else (dz,) * P
        grads_w = [x[:, :K].t() @ g for x, K, g in zip(xs, ctx.Ks, dzs)]           # dW = X^T dZ  (library GEMM)
        # the source rows need dX = dZ W^T: every column for a previous layer, only the embedding columns [0, d) of the
        # layer-0 table (feature columns are not trainable); a part the branch computes itself always needs all of it
        cols = ctx.F_in if ctx.src_needs_grad else ctx.emb_shape[1] if ctx.emb_shape is not None else 0
        dxs = [g @ W.t() if p >= ctx.branch.row_parts else g @ W[:cols].t() if cols else None
               for p, (g, W) in enumerate(zip(dzs, params))]
        grads_own, contribs = ctx.branch.backward(xs, dxs, params[P:], kept, cols)
        dsrc, demb = ctx.branch.source_grads(ctx, contribs, dy)
        return (None, dsrc, demb) + tuple(grads_w) + tuple(grads_own)


def _source_grads(ctx, contribs, dy):
    """contribs: per segment (s, self contribution, neighbour contribution), each (grad rows, group, divisor, dropout site
    or None): row r of s's self (neighbour) rows receives drop(grad[r // group] / divisor).  A layer >= 1 source takes
    them into its row ranges, neighbour rows first, launched in this fixed order so dsrc is reproducible; the layer-0
    embedding table through _embedding_grad, [self, neighbour] lists per segment."""
    dsrc = demb = None
    if ctx.src_needs_grad:
        dsrc = torch.zeros(ctx.src_shape, dtype=dy.dtype, device=dy.device)
        for s, cself, cneigh in contribs:
            if s.self_ids is not None or s.neigh_ids is not None:
                raise NotImplementedError("gradient w.r.t. an id-addressed source (trainable features) is out of scope")
            for row0, rows, (g, group, div, site) in ((s.neigh_row0, s.n * s.k, cneigh), (s.self_row0, s.n, cself)):
                out = dsrc[row0:row0 + rows]
                if site is not None:                    # the mask regenerated
                    ops.dropout_apply(g, site, rows=rows, group=group, scale=1.0 / div, accumulate=True, out=out)
                else:
                    out.view(rows // group, group, ctx.src_shape[1]).add_((g / div if div != 1 else g).unsqueeze(1))
    if ctx.emb_shape is not None:
        d = ctx.emb_shape[1]
        lists, sites = [], []
        for s, cself, cneigh in contribs:
            for ids, rows, (g, group, div, site) in ((s.self_ids, s.n, cself), (s.neigh_ids, s.n * s.k, cneigh)):
                lists.append((ids[:rows], g[:, :d], group, 1.0 / div))
                sites.append(site)                      # entry i of a list is position i of its site
        demb = _embedding_grad(ctx.emb_shape, lists, sites if any(x is not None for x in sites) else None)
    return dsrc, demb


class _AggregateRowsFn(object):
    """The _LayerFn branch of MeanAggregator / GCNAggregator: the fused gather gives the self rows and the fanout mean, or
    for GCN the mean over the k neighbours and the node itself.  sites: None, or one (neighbour site, self site) pair of
    (seed, call, rate) per segment (training dropout): the gather then drops the rows it reads, so the parts are what
    dW = X^T dZ needs."""
    source_grads = staticmethod(_source_grads)

    @staticmethod
    def apply(agg, src, segments, emb, sites, *weights):
        """weights: agg's [weights] (GCN) or [self_weights, neigh_weights]."""
        return _LayerFn.apply(_AggregateRowsFn(agg, segments, sites), src, emb, *weights)

    def __init__(self, agg, segments, sites):
        self.agg, self.segments, self.sites = agg, segments, sites
        self.gcn = "weights" in agg.vars
        self.row_parts = 1 if self.gcn else 2

    def forward(self, src, kept):
        if self.sites is not None:
            ns, ss = [p[0] for p in self.sites], [p[1] for p in self.sites]
            xs, xm = ops.gather_mean_dropout(src, self.segments, ns, ss, include_self=self.gcn, want_self=not self.gcn)
        else:
            xs, xm = ops.gather_mean(src, self.segments, include_self=self.gcn, want_self=not self.gcn)
        F_in, v = src.shape[1], self.agg.vars
        if self.gcn:
            return [(xm, F_in, v["weights"])]
        return [(xs, F_in, v["self_weights"]), (xm, F_in, v["neigh_weights"])]

    def backward(self, xs, dxs, params, kept, cols):
        if not cols:
            return [], []
        dxm = dxs[-1]
        contribs = []
        for i, s in enumerate(self.segments):
            rows = slice(s.out_row0, s.out_row0 + s.n)
            nsite, ssite = self.sites[i] if self.sites is not None else (None, None)
            div = float(s.k + (1 if self.gcn else 0))   # gcn: every row of the mean over [neighbours, self] gets dxm / (k + 1)
            cself = (dxm[rows], 1, div, ssite) if self.gcn else (dxs[0][rows], 1, 1, ssite)
            contribs.append((s, cself, (dxm[rows], s.k, div, nsite)))
        return [], contribs


class _SummaryBranch(object):
    """The _LayerFn branches of the pools and seq: parts [self rows, per-hop neighbour summary]; the self rows receive
    dZ_s Ws^T.  Their apply takes agg's self_weights, neigh_weights and the two tensors of the summary's own layer."""
    row_parts = 1
    source_grads = staticmethod(_source_grads)

    def __init__(self, agg, segments):
        self.agg, self.segments = agg, segments

    def _contribs(self, dxs, neigh_grads):
        return [(s, (dxs[s.out_row0:s.out_row0 + s.n], 1, 1, None), (g, 1, 1, None))
                for s, g in zip(self.segments, neigh_grads)]


class _PoolAggregateRowsFn(_SummaryBranch):
    """MaxPoolingAggregator / MeanPoolingAggregator / TwoMaxLayerPoolingAggregator, materialised on the fp32 kernels:
    gather -> the chain of Dense(relu, bias) layers -> pool over the fanout, keeping per hop each Dense layer's input and
    the last one's output.  The last Dense goes back through pool_branch_backward, the ones before it through
    dpre = dh * [h > 0], dW = x^T dpre, db = sum dpre, dx = dpre W^T.  sites: None, or per segment the dropout site of
    each Dense layer's input - one (seed, call, rate) with one Dense, a (mlp, mlp2) pair with two (training dropout,
    layers.py:107; the self rows are not dropped); the kept inputs are the dropped ones, which is what dW = x^T dpre
    needs, and a dropped zero has no gradient, so [x > 0] of the kept input is the ReLU mask."""

    @staticmethod
    def apply(agg, src, segments, Ws, Wn, *rest):
        """rest: (weights, bias) of each Dense layer in order, then optionally emb and sites."""
        n = 2 * len(agg.mlp_layers)
        emb, sites = (tuple(rest[n:]) + (None, None))[:2]
        return _LayerFn.apply(_PoolAggregateRowsFn(agg, segments, sites), src, emb, Ws, Wn, *rest[:n])

    def __init__(self, agg, segments, sites):
        _SummaryBranch.__init__(self, agg, segments)
        self.sites = sites

    def forward(self, src, kept):
        if len(self.agg.mlp_layers) not in (1, 2) or self.agg.dropout:
            raise NotImplementedError("training supports one or two MLP layers and dropout = 0")
        self.F_in = src.shape[1]
        return self.agg._pooled_parts(src, self.segments, kept, self.sites)

    def backward(self, xs, dxs, params, kept, cols):
        hp, dhp, L = xs[1], dxs[1], len(self.agg.mlp_layers)
        grads = []
        for W in params[0::2]:
            grads += [torch.zeros_like(W), torch.zeros(W.shape[1], dtype=dhp.dtype, device=dhp.device)]
        dxn_all = []
        for i, s in enumerate(self.segments):
            rows = slice(s.out_row0, s.out_row0 + s.n)
            ins, h = list(kept[(L + 1) * i:(L + 1) * i + L]), kept[(L + 1) * i + L]
            ins[0] = ins[0][:, :self.F_in]
            hop_sites = None if self.sites is None else (self.sites[i],) if L == 1 else self.sites[i]
            W = params[2 * L - 2]
            g_w, g_b, dx = pool_branch_backward(self.agg.pool, ins[-1], h, hp[rows], dhp[rows], W[:cols] if L == 1 else W,
                                                s.k, L > 1 or cols > 0)
            grads[2 * L - 2] += g_w
            grads[2 * L - 1] += g_b
            for j in range(L - 2, -1, -1):                    # the Dense layers before the last, through their ReLU
                if hop_sites is not None:                     # the input mask of Dense j + 1, regenerated
                    dx = ops.dropout_apply(dx, hop_sites[j + 1])
                dpre = dx * (ins[j + 1] > 0).to(dx.dtype)
                grads[2 * j] += ins[j].t() @ dpre
                grads[2 * j + 1] += dpre.sum(dim=0)
                W = params[2 * j]
                dx = (dpre @ (W[:cols] if j == 0 else W).t()) if (j > 0 or cols) else None
            if dx is not None and hop_sites is not None:      # through the input mask, regenerated
                dx = ops.dropout_apply(dx, hop_sites[0])
            dxn_all.append(dx)
        return grads, (self._contribs(dxs[0], dxn_all) if cols else [])


def refuse_fused_pool(model):
    """The limits of the fused bf16 pooling branch (fused_pool=True) that are known once the aggregators exist."""
    if not getattr(model, "fused_pool", False):
        return
    if not hasattr(model.aggregators[0], "mlp_layers"):
        raise NotImplementedError("fused_pool=True applies to the maxpool and meanpool aggregators only")
    refuse_int8_table(model.features, "fused_pool=True")
    if hasattr(model.features, "c_table"):
        raise NotImplementedError("fused_pool=True with a node-partitioned (ShardedFeatures) table is not implemented")
    if model.dropout_rate:
        raise NotImplementedError("fused_pool=True with training dropout > 0 is not implemented (the MLP input would "
                                  "have to be masked inside K4)")
    for info in model.layer_infos:
        if info.num_samples > FUSED_POOL_MAX_FANOUT:
            raise NotImplementedError("fused_pool=True needs fanouts <= %d (got %d)" % (FUSED_POOL_MAX_FANOUT, info.num_samples))
    for agg in model.aggregators:
        if agg.neigh_input_dim > FUSED_POOL_MAX_K:
            raise NotImplementedError("fused_pool=True needs layer input widths <= %d (got %d)"
                                      % (FUSED_POOL_MAX_K, agg.neigh_input_dim))
        if agg.hidden_dim % FUSED_POOL_HIDDEN_STEP != 0:
            raise NotImplementedError("fused_pool=True needs a pooling hidden width that is a multiple of %d (got %d)"
                                      % (FUSED_POOL_HIDDEN_STEP, agg.hidden_dim))
        if len(agg.mlp_layers) != 1:
            raise NotImplementedError("fused_pool=True supports one MLP layer")


class _FusedPoolAggregateRowsFn(_SummaryBranch):
    """MaxPoolingAggregator / MeanPoolingAggregator through the fused bf16 kernels (fused_pool=True): K4
    (ops.maxpool_mlp_fused) in the forward; the backward recomputes the MLP tile instead of storing it (B1
    ops.pool_mlp_backward_dp), then dWm / dbm (B2) and, where a source gradient is needed, dX (B3).  bf16 operands with
    fp32 accumulation whatever agg.math is.  Kept: the bf16 operand table - neither the gathered neighbour rows nor the
    MLP activations.  persistent: src is the model's feature table (layer 0), cast to bf16 once per table version; a
    layer >= 1 source is cast on every call."""

    @staticmethod
    def apply(agg, src, segments, Ws, Wn, Wm, bm, emb=None, persistent=False):
        return _LayerFn.apply(_FusedPoolAggregateRowsFn(agg, segments, persistent), src, emb, Ws, Wn, Wm, bm)

    def __init__(self, agg, segments, persistent):
        _SummaryBranch.__init__(self, agg, segments)
        self.persistent = persistent

    def forward(self, src, kept):
        agg = self.agg
        if hasattr(src, "c_table"):
            raise NotImplementedError("fused_pool=True with a node-partitioned (ShardedFeatures) table is not implemented")
        F_in, hid = src.shape[1], agg.hidden_dim
        for s in self.segments:
            if not fused_pool_fits(s.k, F_in, hid):
                raise NotImplementedError("fused_pool=True needs fanout <= %d, input width <= %d and hidden %% %d == 0 "
                                          "(k=%d K=%d hidden=%d)" % (FUSED_POOL_MAX_FANOUT, FUSED_POOL_MAX_K,
                                                                     FUSED_POOL_HIDDEN_STEP, s.k, F_in, hid))
        self.F_in = F_in
        table = agg._bf16_table(src, self.persistent)
        kept.append(table)
        return agg._summarise(src, self.segments, lambda i, s, out: agg._fused_hop(table, s, out), f32_self=True)

    def backward(self, xs, dxs, params, kept, cols):
        (Wm, bm), dhp, (table,), agg = params, dxs[1], kept, self.agg
        dWm, dbm = torch.zeros_like(Wm), torch.zeros(Wm.shape[1], dtype=dhp.dtype, device=dhp.device)
        if cols and (getattr(agg, "_packed_dx", None) is None or agg._packed_dx.cols != cols):
            agg._packed_dx = ops.PackedMlpDxWeights(cols)
        dxn_all = []
        for s in self.segments:                               # per hop, in order: B1 -> B2 (dWm, dbm) -> B3
            n, k = s.n, s.k
            grad = ops.pool_mlp_backward_dp(table, n, k, Wm, bm, agg._packed_mlp, dhp[s.out_row0:s.out_row0 + n],
                                            row_ids=s.neigh_ids, row0=s.neigh_row0, K=self.F_in, pool=agg.pool)
            ops.pool_mlp_backward_dw(table, n, k, grad, dWm, dbm, row_ids=s.neigh_ids, row0=s.neigh_row0, K=self.F_in)
            if cols:
                dxn_all.append(ops.pool_mlp_backward_dx(grad, n, k, Wm, agg._packed_dx))
        return [dWm, dbm], (self._contribs(dxs[0], dxn_all) if cols else [])


class _SeqAggregateRowsFn(_SummaryBranch):
    """SeqAggregator.  Forward per hop: X (gathered rows, or the previous layer's row range) -> lengths (gs_seq_lengths)
    -> P = X W_x + b (library GEMM, agg.math) -> gs_lstm_forward, keeping X, the lengths, the gates, c and h_{t-1}.
    Backward per hop: gs_lstm_backward gives dZ; dW_x = X^T dZ, dW_h = h_prev^T dZ, db = sum dZ and dX = dZ W_x^T are
    library matmuls."""

    @staticmethod
    def apply(agg, src, segments, Ws, Wn, kernel, cell_bias, emb=None):
        return _LayerFn.apply(_SeqAggregateRowsFn(agg, segments), src, emb, Ws, Wn, kernel, cell_bias)

    def forward(self, src, kept):
        self.F_in = src.shape[1]
        return self.agg._seq_parts(src, self.segments, kept)

    def backward(self, xs, dxs, params, kept, cols):
        kernel, dhl = params[0], dxs[1]
        Wx, Wh = kernel[:self.F_in], kernel[self.F_in:]
        dWx, dWh = torch.zeros_like(Wx), torch.zeros_like(Wh)
        db = torch.zeros(kernel.shape[1], dtype=dhl.dtype, device=dhl.device)
        dX_all = []
        for i, s in enumerate(self.segments):
            X, lengths, gates, c, h_prev = kept[5 * i:5 * i + 5]
            dZ = ops.lstm_backward(dhl[s.out_row0:s.out_row0 + s.n], gates, c, lengths, Wh, s.n, s.k)
            dWx += X.t() @ dZ
            dWh += h_prev.t() @ dZ
            db += dZ.sum(dim=0)
            if cols:
                dX_all.append(dZ @ Wx[:cols].t())
        return [torch.cat([dWx, dWh]), db], (self._contribs(dxs[0], dX_all) if cols else [])


def layer_params(agg):
    """The tensors a layer trains, in _LayerFn's order: the GEMM parts' weights ([weights] for GCN, else [self_weights,
    neigh_weights]), then the branch's own - each of the pools' Dense layers' weights and bias, the seq cell's kernel and
    bias."""
    v = agg.vars
    if hasattr(agg, "cell"):
        cell = agg.cell.vars
        return v["self_weights"], v["neigh_weights"], cell["kernel"], cell["bias"]
    if hasattr(agg, "mlp_layers"):
        if len(agg.mlp_layers) != 1 and not isinstance(agg, TwoMaxLayerPoolingAggregator):
            raise NotImplementedError("training supports one MLP layer")
        return (v["self_weights"], v["neigh_weights"]) + tuple(
            t for layer in agg.mlp_layers for t in (layer.vars["weights"], layer.vars["bias"]))
    return (v["weights"],) if "weights" in v else (v["self_weights"], v["neigh_weights"])


def train_layer(agg, src, segments, emb=None, sites=None, fused=False, persistent=False):
    """agg.aggregate_rows(src, segments) with an autograd graph (_LayerFn): through the seq, the materialised or (fused)
    the fused bf16 pooling branch, or the mean / GCN one.  sites: training dropout of the mean / GCN and materialised
    pooling branches (see their classes); persistent: src is the model's layer-0 feature table."""
    params = layer_params(agg)
    if hasattr(agg, "cell"):
        return _SeqAggregateRowsFn.apply(agg, src, segments, *params, emb)
    if hasattr(agg, "mlp_layers"):
        fn, extra = (_FusedPoolAggregateRowsFn, persistent) if fused else (_PoolAggregateRowsFn, sites)
        return fn.apply(agg, src, segments, *params, emb, extra)
    return _AggregateRowsFn.apply(agg, src, segments, emb, sites, *params)


def differentiable_outputs(model, batch, normalize=True, dropout=0.):
    """sample -> aggregate (-> l2_normalize) with an autograd graph over the aggregator weights; `model` is a
    SampleAndAggregate whose .aggregators exist (reference models.py:347-350 / supervised_models.py:79-85).
    dropout = p > 0: training dropout, sites numbered by dropout_site_plan from model.dropout_counter, which advances
    past them (p = 0 draws nothing and leaves the counter alone); model.dropout_call_dev, when set, is the device-side
    offset every site adds to its call number (graphed_training)."""
    dropout = check_dropout_rate(dropout)
    fused = getattr(model, "fused_pool", False)
    if dropout:
        if fused:
            raise NotImplementedError("fused_pool=True with training dropout > 0 is not implemented (the MLP input would "
                                      "have to be masked inside K4)")
        refuse_dropout_table(model.features)
    batch = batch.to(device=model.device, dtype=torch.int32).reshape(-1)
    n = batch.numel()
    with torch.no_grad():
        samples, support = model.sample(batch, model.layer_infos, batch_size=n)
    num_samples = [info.num_samples for info in model.layer_infos]
    L = len(num_samples)
    counts = [n * support[h] for h in range(L + 1)]
    # a host table's layer-0 source is this step's working set, rewritten by the next stage: never the cached bf16 cast
    src, samples, persistent = stage_layer0(model.features, samples)
    pool = hasattr(model.aggregators[0], "mlp_layers")
    two = isinstance(model.aggregators[0], TwoMaxLayerPoolingAggregator)
    seq = hasattr(model.aggregators[0], "cell")
    kind = "seq" if seq else "twomaxpool" if two else "maxpool" if pool else "mean"
    plan = dropout_site_plan(kind, L) if dropout else []
    call = {site: model.dropout_counter + i for i, site in enumerate(plan)}
    for layer in range(L):
        hops = L - layer
        # layer 0 reads the embedding table (identity_dim > 0) through src; handing it over as an input lets autograd
        # deliver the scattered gradient as embeds.grad
        emb = getattr(model, "embeds", None) if layer == 0 else None
        sites = None
        if dropout and not seq:                              # per hop: the MLP-input site, or the (neighbour, self) pair
            key, dev = model.dropout_key, model.dropout_call_dev
            if two:                                          # the inputs of both Dense layers
                sites = [tuple((key, call[(layer, h, role)], dropout, dev) for role in ("mlp", "mlp2"))
                         for h in range(hops)]
            elif pool:
                sites = [(key, call[(layer, h, "mlp")], dropout, dev) for h in range(hops)]
            else:
                sites = [((key, call[(layer, h, "neigh")], dropout, dev), (key, call[(layer, h, "self")], dropout, dev))
                         for h in range(hops)]
        src = train_layer(model.aggregators[layer], src, layer_segments(samples, counts, num_samples, layer), emb, sites,
                          fused, layer == 0 and persistent)
    model.dropout_counter += len(plan)
    out = src[:counts[0]]
    if normalize:
        out = out / torch.sqrt(torch.clamp((out * out).sum(dim=1, keepdim=True), min=1e-12))   # tf.nn.l2_normalize
    return out


def check_dropout_rate(rate):
    rate = float(rate or 0.)
    if not 0.0 <= rate < 1.0:
        raise ValueError("dropout must be in [0, 1) (got %r)" % (rate,))
    return rate


def refuse_dropout_table(features):
    """Training dropout needs the dense fp32 table of the masked gather kernel."""
    if hasattr(features, "c_table"):
        raise NotImplementedError("training dropout with a node-partitioned (ShardedFeatures) table is not implemented")
    if features.dtype != torch.float32:
        raise NotImplementedError("training dropout with a %s feature table is not implemented (float32 only)"
                                  % features.dtype)


def init_dropout(model, dropout_seed, distributed, group):
    """The training rate placeholders['dropout'] (validated), the mask key and the site counter.  With distributed=True
    the key is dropout_seed + rank, so the ranks draw independent masks for their different batches."""
    rate = check_dropout_rate(model.placeholders.get("dropout", 0.))
    if rate:
        refuse_dropout_table(model.features)
    key = int(dropout_seed)
    if distributed:
        import torch.distributed as dist
        key += dist.get_rank(group)
    model.dropout_rate, model.dropout_key, model.dropout_counter = rate, key, 0
    model.dropout_call_dev = None       # device offset of every call number, set while a training step is captured


def build_aggregators(model):
    """One aggregator per layer, as SampleAndAggregate.aggregate creates them (reference models.py:303-315).  Their own
    .dropout stays 0 - forward, graphed, pipelined and export paths keep the fused inference kernels; the training rate
    placeholders['dropout'] is applied by the training pass (differentiable_outputs)."""
    L = len(model.layer_infos)
    aggs = []
    for layer in range(L):
        dim_mult = 2 if model.concat and layer != 0 else 1
        act = identity if layer == L - 1 else relu
        extra = {"model_size": model.model_size} if issubclass(model.aggregator_cls, _SIZED_AGGREGATORS) else {}
        aggs.append(model.aggregator_cls(dim_mult * model.dims[layer], model.dims[layer + 1], act=act, dropout=0.,
                                         concat=model.concat, device=model.device, **extra))
    return aggs


def aggregator_parameters(aggregators):
    """(all trainable tensors, the subset the reference applies weight decay to).  The reference decays
    `aggregator.vars` only (supervised_models.py:103-105, models.py:385-387) - the pooling aggregators' Dense variables
    live in `mlp_layers[0].vars` and the seq aggregator's LSTM kernel and bias in `cell.vars`: both are trained but not
    decayed."""
    decayed = [v for a in aggregators for v in a.vars.values()]
    extra = [v for a in aggregators for layer in getattr(a, "mlp_layers", []) for v in layer.vars.values()]
    extra += [v for a in aggregators if hasattr(a, "cell") for v in a.cell.vars.values()]
    return decayed + extra, decayed


def embedding_parameters(model):
    """[model.embeds] when the model trains node embeddings (identity_dim > 0), else [].  Trained and clipped with the
    rest, never weight-decayed (the reference decays aggregator and head variables only)."""
    return [model.embeds] if getattr(model, "embeds", None) is not None else []


def refuse_distributed_host_table(features, distributed):
    if distributed:
        refuse_host_table(features, "distributed=True")
        refuse_int8_table(features, "distributed=True")


def refuse_distributed_embeddings(identity_dim, distributed):
    if identity_dim > 0 and distributed:
        raise NotImplementedError("identity_dim > 0 with distributed=True is not implemented (the [N+1, d] table would "
                                  "have to be sharded or its dense gradient all-reduced)")


def classification_loss(logits, labels, sigmoid_loss):
    """reference supervised_models.py:109-117: mean over ALL elements of the sigmoid cross-entropy (multi-label), or the
    mean over nodes of the softmax cross-entropy."""
    if sigmoid_loss:
        return torch.nn.functional.binary_cross_entropy_with_logits(logits, labels, reduction="mean")
    return (-(labels * torch.log_softmax(logits, dim=1)).sum(dim=1)).mean()


def weight_decay_term(params, weight_decay):
    """weight_decay * tf.nn.l2_loss(var) = weight_decay * sum(var^2) / 2 over every variable (supervised_models.py:103-107)."""
    total = None
    for p in params:
        t = weight_decay * 0.5 * (p * p).sum()
        total = t if total is None else total + t
    return total


def clipped_step(model, loss):
    """One optimiser step of the supervised and unsupervised models on `loss`: gradients, their mean over the ranks when
    model.distributed (data parallel), clip_by_value(grad, -5, 5) (supervised_models.py:93-94, models.py:380-381), Adam.
    Returns the detached loss."""
    model.optimizer.zero_grad(set_to_none=True)
    loss.backward()
    if model.distributed:
        from .parallel import allreduce_gradients
        model.last_allreduce_bytes = allreduce_gradients(model.parameters(), model.group)
    for p in model.parameters():
        if p.grad is not None:
            p.grad.clamp_(-5.0, 5.0)
    model.optimizer.step()
    return loss.detach()


class SupervisedGraphsage(SampleAndAggregate):
    """Supervised GraphSAGE (reference graphsage/supervised_models.py:10-126): the hot path, then
    l2_normalize -> Dense(-> num_classes) -> sigmoid / softmax cross-entropy (+ weight decay), gradients clipped to
    [-5, 5], Adam.  TF FLAGS become constructor arguments (learning_rate, weight_decay)."""

    def __init__(self, num_classes, placeholders, features, adj, degrees, layer_infos, concat=True,
                 aggregator_type="mean", model_size="small", sigmoid_loss=False, identity_dim=0, learning_rate=0.01,
                 weight_decay=0.0, device="cuda", distributed=False, group=None, dropout_seed=12345, fused_pool=False,
                 **kwargs):
        """dropout_seed: key of the training dropout masks (placeholders['dropout'] > 0); with distributed=True each rank
        uses dropout_seed + rank.  fused_pool: train the maxpool / meanpool branch through the fused bf16 kernels
        (_FusedPoolAggregateRowsFn) instead of the materialised fp32 path."""
        refuse_distributed_embeddings(identity_dim, distributed)
        refuse_distributed_host_table(features, distributed)
        super(SupervisedGraphsage, self).__init__(placeholders, features, adj, degrees, layer_infos, concat=concat,
                                                  aggregator_type=aggregator_type, model_size=model_size,
                                                  identity_dim=identity_dim, device=device, **kwargs)
        if aggregator_type not in ("mean", "gcn", "maxpool", "meanpool", "twomaxpool", "seq"):
            raise NotImplementedError("training is implemented for the mean, gcn, maxpool, meanpool, twomaxpool and seq "
                                      "aggregators")
        init_dropout(self, dropout_seed, distributed, group)
        self.num_classes = num_classes
        self.sigmoid_loss = sigmoid_loss
        self.learning_rate, self.weight_decay = learning_rate, weight_decay
        self.distributed, self.group, self.last_allreduce_bytes = bool(distributed), group, 0
        self.fused_pool = bool(fused_pool)
        self.build()
        refuse_fused_pool(self)

    def build(self):
        from .inits import glorot, zeros
        self.aggregators = build_aggregators(self)
        dim_mult = 2 if self.concat else 1
        self.node_pred_vars = {"weights": glorot([dim_mult * self.dims[-1], self.num_classes], device=self.device),
                               "bias": zeros([self.num_classes], device=self.device)}   # supervised_models.py:88-90
        if self.distributed:                                                     # every rank starts from rank 0's weights
            from .parallel import broadcast_parameters
            broadcast_parameters(self.parameters(), 0, self.group)
        for p in self.parameters():
            p.requires_grad_(True)
        self.optimizer = torch.optim.Adam(self.parameters(), lr=self.learning_rate)      # TF AdamOptimizer defaults

    def parameters(self):
        return aggregator_parameters(self.aggregators)[0] + list(self.node_pred_vars.values()) + embedding_parameters(self)

    def decayed_parameters(self):
        return aggregator_parameters(self.aggregators)[1] + list(self.node_pred_vars.values())

    def outputs(self, batch, dropout=0.):
        """l2-normalised node representations, differentiable (supervised_models.py:79-85).  dropout: the training
        rate (0 = the reference's evaluation default, placeholder_with_default(0.))."""
        return differentiable_outputs(self, batch, dropout=dropout)

    def logits(self, batch, dropout=0.):
        """node_pred(outputs) (supervised_models.py:88-92); with dropout > 0 the head input is dropped too (one more
        site, after the aggregators')."""
        out = self.outputs(batch, dropout=dropout)
        if check_dropout_rate(dropout):
            out = _DropoutFn.apply(out, (self.dropout_key, self.dropout_counter, dropout, self.dropout_call_dev))
            self.dropout_counter += 1
        return self._node_pred(out)

    def _node_pred(self, out):
        return out @ self.node_pred_vars["weights"] + self.node_pred_vars["bias"]

    def loss(self, batch, labels, dropout=0.):
        """supervised_models.py:101-118: weight decay * l2_loss(var) over aggregator + head variables, then the
        mean of the per-element sigmoid xent (multi-label) or the mean of the per-node softmax xent."""
        logits = self.logits(batch, dropout=dropout) if dropout else self.logits(batch)    # overrides take (batch)
        return self._logits_loss(logits, labels)

    def _logits_loss(self, logits, labels):
        """loss()'s tail on the head's logits, shared with the full-neighbourhood losses."""
        self._last_logits = logits.detach()
        labels = torch.as_tensor(labels).to(device=logits.device, dtype=torch.float32)
        loss = classification_loss(logits, labels, self.sigmoid_loss)
        if self.weight_decay:
            loss = loss + weight_decay_term(self.decayed_parameters(), self.weight_decay)
        return loss

    def train_step(self, batch, labels):
        """One Adam step at the training dropout rate placeholders['dropout'] (supervised_train.py:271)."""
        return clipped_step(self, self.loss(batch, labels, dropout=self.dropout_rate))

    def graphed_train_step(self, batch_size):
        """train_step for a fixed batch size captured in one CUDA graph: returns step(batch, labels) -> loss, a static 0-d
        CUDA tensor (see graphed_training.GraphedTrainStep; a short last batch runs through the eager train_step)."""
        return GraphedTrainStep(self, batch_size)

    def predict(self, batch):
        with torch.no_grad():
            return self._predictions(self.logits(batch))

    def full_neighbor_outputs(self, indptr, indices, node_ids, dropout=None, edge_weight=None):
        """outputs() over whole neighbourhoods: full_neighbor_embeddings(indptr, indices, node_ids) - the same bits -
        with an autograd graph over the aggregator weights and (identity_dim > 0) the node embeddings, for any head to
        compose (contract: oracle/full_neighbor_grad.py).  The CSR's transposes are built on first use and cached on the
        model, keyed by the CSR tensors' data_ptr, numel and _version.  dropout: None (no masks), or a training rate
        p in [0, 1) - callers pass dropout=model.dropout_rate.  The full-neighbourhood masks follow their own contract
        (one per CSR entry and per node, keyed by global ids: oracle/full_neighbor_dropout.py), not the sampled one, so
        they are applied only when asked for; p = 0 gives the bits of dropout=None.  Refused (NotImplementedError): the
        seq aggregator, ShardedFeatures, distributed=True, CUDA-graph capture, and dropout=None on a model whose
        dropout_rate > 0.  edge_weight: as full_neighbor_embeddings (weighted messages, oracle/weighted.py); the
        transposes' weights are cached with the transposes, keyed by the weight tensor too.  Refused with dropout p > 0."""
        from .full_neighbor_training import full_neighbor_outputs
        return full_neighbor_outputs(self, indptr, indices, node_ids, dropout=dropout, edge_weight=edge_weight)

    def _full_neighbor_logits(self, out, dropout):
        """The head on full-neighbourhood outputs; with p > 0 its input is dropped at the site after the layers'."""
        p = check_full_neighbor_dropout(dropout)
        if p:
            out = _DropoutFn.apply(out, (self.dropout_key, self.dropout_counter, p, None))
            self.dropout_counter += 1
        return self._node_pred(out)

    def full_neighbor_loss(self, indptr, indices, node_ids, labels, dropout=None, edge_weight=None):
        """loss() on full_neighbor_outputs: the same head, cross-entropy and weight decay, over the rows of node_ids.
        dropout: as full_neighbor_outputs; p > 0 also drops the head input (row r of node_ids at position r)."""
        check_full_neighbor_dropout(dropout)
        out = self.full_neighbor_outputs(indptr, indices, node_ids, dropout=dropout, edge_weight=edge_weight)
        return self._logits_loss(self._full_neighbor_logits(out, dropout), labels)

    def full_neighbor_train_step(self, indptr, indices, node_ids, labels, dropout=None, edge_weight=None):
        """One deterministic full-batch Adam step: every node of node_ids over its whole neighbourhood (no sampling;
        dropout as full_neighbor_loss), gradients clipped to +-5 as in train_step.  Returns the detached loss; no host
        synchronisation."""
        return clipped_step(self, self.full_neighbor_loss(indptr, indices, node_ids, labels, dropout=dropout,
                                                          edge_weight=edge_weight))

    def full_neighbor_minibatch_outputs(self, indptr, indices, node_ids, dropout=None, edge_weight=None):
        """full_neighbor_outputs over the receptive field of node_ids only: the same values, bit for bit, with per-layer
        blocks built on the device by ops.csr_blocks (contract: oracle/full_neighbor_blocks.py) and their transposes built
        per call, not cached.  Cost and memory follow the blocks, not the graph: the minibatch form of exact-neighbourhood
        training.  Reads the block sizes back once per call.  dropout and refusals as full_neighbor_outputs: the masks are
        keyed by global ids, so the rows equal the whole-graph pass's from the same counter.  edge_weight: as
        full_neighbor_outputs, each block entry carrying its raw CSR entry's weight (built per call)."""
        from .full_neighbor_training import full_neighbor_outputs
        return full_neighbor_outputs(self, indptr, indices, node_ids, minibatch=True, dropout=dropout,
                                     edge_weight=edge_weight)

    def full_neighbor_minibatch_loss(self, indptr, indices, node_ids, labels, dropout=None, edge_weight=None):
        """full_neighbor_loss over full_neighbor_minibatch_outputs: the same head, cross-entropy and weight decay."""
        check_full_neighbor_dropout(dropout)
        out = self.full_neighbor_minibatch_outputs(indptr, indices, node_ids, dropout=dropout, edge_weight=edge_weight)
        return self._logits_loss(self._full_neighbor_logits(out, dropout), labels)

    def full_neighbor_minibatch_train_step(self, indptr, indices, node_ids, labels, dropout=None, edge_weight=None):
        """full_neighbor_train_step for a minibatch: one Adam step on full_neighbor_minibatch_loss, gradients clipped to
        +-5.  Returns the detached loss."""
        return clipped_step(self, self.full_neighbor_minibatch_loss(indptr, indices, node_ids, labels, dropout=dropout,
                                                                    edge_weight=edge_weight))

    def sampled_minibatch_outputs(self, indptr, indices, node_ids, dropout=None, edge_weight=None, sample_weight=None):
        """outputs() over sampled receptive-field blocks (SampleAndAggregate.sampled_minibatch_embeddings; contract:
        oracle/sampled_blocks.py), with an autograd graph over the aggregator weights and (identity_dim > 0) the node
        embeddings.  One block set per call: the sampler's counter advances by 1.  dropout: None (no masks), or a
        training rate p in [0, 1) - callers pass dropout=model.dropout_rate: the full-neighbourhood masks, a sampled
        entry masked as the same CSR entry is in the whole-graph pass (contract: oracle/sampled_blocks_dropout.py), sites
        numbered from dropout_counter; p = 0 gives the bits of dropout=None.  Refused (NotImplementedError): what
        full_neighbor_outputs refuses but host-memory and int8 tables (taken here: see sampled_minibatch_embeddings),
        CUDA-graph capture, dropout=None on a model whose dropout_rate > 0, and dropout = p > 0 on an int8 table.
        edge_weight: as full_neighbor_outputs, each sampled entry carrying its raw CSR entry's weight; refused with
        dropout p > 0.  sample_weight: as sampled_minibatch_embeddings, the blocks drawn in proportion to it; it
        combines with edge_weight and with dropout."""
        from .full_neighbor_training import full_neighbor_outputs
        return full_neighbor_outputs(self, indptr, indices, node_ids, minibatch=True, sampled=True, dropout=dropout,
                                     edge_weight=edge_weight, sample_weight=sample_weight)

    def sampled_minibatch_loss(self, indptr, indices, node_ids, labels, dropout=None, edge_weight=None,
                               sample_weight=None):
        """loss() over sampled_minibatch_outputs: the same head, cross-entropy and weight decay.  dropout: as
        sampled_minibatch_outputs; p > 0 also drops the head input (row r of node_ids at position r).  sample_weight: as
        sampled_minibatch_outputs."""
        check_full_neighbor_dropout(dropout)
        out = self.sampled_minibatch_outputs(indptr, indices, node_ids, dropout=dropout, edge_weight=edge_weight,
                                             sample_weight=sample_weight)
        return self._logits_loss(self._full_neighbor_logits(out, dropout), labels)

    def sampled_minibatch_train_step(self, indptr, indices, node_ids, labels, dropout=None, edge_weight=None,
                                     sample_weight=None):
        """One Adam step on sampled_minibatch_loss, gradients clipped to +-5 as in train_step.  Returns the detached
        loss."""
        return clipped_step(self, self.sampled_minibatch_loss(indptr, indices, node_ids, labels, dropout=dropout,
                                                              edge_weight=edge_weight, sample_weight=sample_weight))

    def full_neighbor_predict(self, indptr, indices, node_ids, edge_weight=None):
        """predict() over whole neighbourhoods: the head (supervised_models.py:88-92, 120-126) on
        full_neighbor_embeddings(indptr, indices, node_ids, edge_weight=edge_weight) - deterministic, no sampling, no
        dropout."""
        with torch.no_grad():
            return self._predictions(self._node_pred(self.full_neighbor_embeddings(indptr, indices, node_ids,
                                                                                   edge_weight=edge_weight)))

    def last_predictions(self):
        """model.preds of the last loss() / train_step() call (supervised_models.py:120-126): the predictions from that
        call's own logits - before its update, at its dropout rate - without another forward pass (which would draw new
        samples and masks).  After a replay of graphed_train_step, the replay's."""
        with torch.no_grad():
            return self._predictions(self._last_logits)

    def _predictions(self, logits):
        return torch.sigmoid(logits) if self.sigmoid_loss else torch.softmax(logits, dim=1)
