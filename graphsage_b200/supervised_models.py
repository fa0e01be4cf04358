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
from .layers import act_code, identity, relu  # noqa: F401
from .aggregators import refuse_seq_table
from .models import _SIZED_AGGREGATORS, SampleAndAggregate


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
    for layer in range(n_layers):
        for hop in range(n_layers - layer):
            plan += [(layer, hop, "mlp")] if kind in ("maxpool", "meanpool") else [(layer, hop, "neigh"), (layer, hop, "self")]
    return plan + ([(None, None, "head")] if head else [])


class _DropoutFn(torch.autograd.Function):
    """y = drop(x) for one site (the supervised head's input, layers.py:107); the backward applies the same mask."""

    @staticmethod
    def forward(ctx, x, site):
        ctx.site = site
        return ops.dropout_apply(x.detach(), site)

    @staticmethod
    def backward(ctx, dy):
        return ops.dropout_apply(dy.contiguous(), ctx.site), None


class _AggregateRowsFn(torch.autograd.Function):
    """y = agg.aggregate_rows(src, segments) for MeanAggregator / GCNAggregator, differentiable w.r.t. the
    aggregator weights, (for layers >= 1, where rows are addressed by ranges) w.r.t. src, and (layer 0, identity_dim > 0)
    w.r.t. `emb`, the [N+1, d] embedding view of src's first d columns."""

    @staticmethod
    def forward(ctx, agg, src, segments, emb, sites, *weights):
        """sites: None, or one (neighbour site, self site) pair of (seed, call, rate) per segment (training dropout);
        xs / xm are then the dropped self rows and the mean of the dropped rows, which is what dW = X^T dZ needs."""
        kind = "gcn" if "weights" in agg.vars else "mean"
        code, post = act_code(agg.act)
        if post is not None:
            raise NotImplementedError("training supports act=relu or identity")
        with torch.no_grad():
            if sites is not None:
                ns, ss = [p[0] for p in sites], [p[1] for p in sites]
                xs, xm = ops.gather_mean_dropout(src, segments, ns, ss, include_self=kind == "gcn", want_self=kind == "mean")
            elif kind == "mean":
                xs, xm = ops.gather_mean(src, segments, want_self=True)
            else:
                xs, xm = None, ops.gather_mean(src, segments, include_self=True, want_self=False)[1]
            F_in = src.shape[1]
            if kind == "mean":
                parts = [(xs, F_in, weights[0]), (xm, F_in, weights[1])]
                combine = ops.COMBINE_CONCAT if agg.concat else ops.COMBINE_ADD
            else:
                parts, combine = [(xm, F_in, weights[0])], ops.COMBINE_ADD
            y = ops.sage_gemm(parts, combine=combine, bias=agg.vars.get("bias"), act=code, math=agg.math)
        ctx.kind, ctx.relu, ctx.concat = kind, code == ops.ACT_RELU, bool(agg.concat)
        ctx.segments, ctx.src_shape, ctx.F_in, ctx.sites = segments, tuple(src.shape), F_in, sites
        ctx.src_needs_grad = bool(torch.is_tensor(src) and src.requires_grad)
        ctx.emb_shape = tuple(emb.shape) if emb is not None and emb.requires_grad else None
        ctx.has_bias = "bias" in agg.vars
        ctx.save_for_backward(xm if xs is None else xs, xm, y, *weights)
        return y

    @staticmethod
    def backward(ctx, dy):
        xs, xm, y = ctx.saved_tensors[:3]
        weights = ctx.saved_tensors[3:]
        F_in = ctx.F_in
        dz = dy * (y > 0).to(dy.dtype) if ctx.relu else dy
        grads_w, dsrc = [], None
        if ctx.kind == "mean":
            Ws, Wn = weights
            D = Ws.shape[1]
            dz_s, dz_n = (dz[:, :D], dz[:, D:]) if ctx.concat else (dz, dz)
            grads_w = [xs[:, :F_in].t() @ dz_s, xm[:, :F_in].t() @ dz_n]         # dW = X^T dZ  (library GEMM)
            if ctx.src_needs_grad:
                dxs, dxm = dz_s @ Ws.t(), dz_n @ Wn.t()
        else:
            (W,) = weights
            grads_w = [xm[:, :F_in].t() @ dz]
            if ctx.src_needs_grad:
                dxm = dz @ W.t()
                dxs = None
        if ctx.src_needs_grad:
            dsrc = torch.zeros(ctx.src_shape, dtype=dy.dtype, device=dy.device)
            for si, s in enumerate(ctx.segments):
                if s.self_ids is not None or s.neigh_ids is not None:
                    raise NotImplementedError("gradient w.r.t. an id-addressed source (trainable features) is out of scope")
                n, k = s.n, s.k
                rows = slice(s.out_row0, s.out_row0 + n)
                div = float(k + (1 if ctx.kind == "gcn" else 0))
                if ctx.sites is not None:
                    # the masks regenerated: neighbour row i*k + j gets mask * dxm[i] / div / keep, the self row mask * dxs[i]
                    # (gcn: mask * dxm[i] / div); launched in this fixed order, so dsrc is reproducible
                    nsite, ssite = ctx.sites[si]
                    ops.dropout_apply(dxm[rows], nsite, rows=n * k, group=k, scale=1.0 / div, accumulate=True,
                                      out=dsrc[s.neigh_row0:s.neigh_row0 + n * k])
                    self_g, self_scale = (dxm[rows], 1.0 / div) if ctx.kind == "gcn" else (dxs[rows], 1.0)
                    ops.dropout_apply(self_g, ssite, scale=self_scale, accumulate=True, out=dsrc[s.self_row0:s.self_row0 + n])
                    continue
                dsrc[s.neigh_row0:s.neigh_row0 + n * k].view(n, k, -1).add_((dxm[rows] / div).unsqueeze(1))
                if ctx.kind == "gcn":
                    dsrc[s.self_row0:s.self_row0 + n].add_(dxm[rows] / div)
                else:
                    dsrc[s.self_row0:s.self_row0 + n].add_(dxs[rows])
        demb = None
        if ctx.emb_shape is not None:
            d = ctx.emb_shape[1]
            # the source gradient restricted to the embedding columns: dZ @ W[:d]^T (feature columns are not trainable)
            if ctx.kind == "mean":
                es, em = dz_s @ weights[0][:d].t(), dz_n @ weights[1][:d].t()
            else:
                es, em = None, dz @ weights[0][:d].t()
            lists, sites = [], ([] if ctx.sites is not None else None)
            for si, s in enumerate(ctx.segments):
                n, k = s.n, s.k
                rows = slice(s.out_row0, s.out_row0 + n)
                if ctx.kind == "gcn":                       # mean over [neighbours, self]: every id gets dxm / (k + 1)
                    lists += [(s.self_ids[:n], em[rows], 1, 1.0 / (k + 1)), (s.neigh_ids[:n * k], em[rows], k, 1.0 / (k + 1))]
                else:                                       # self id: dxs; neighbour ids: dxm / k
                    lists += [(s.self_ids[:n], es[rows], 1, 1.0), (s.neigh_ids[:n * k], em[rows], k, 1.0 / k)]
                if sites is not None:                       # entry i of a list is position i of its site
                    sites += [ctx.sites[si][1], ctx.sites[si][0]]
            demb = _embedding_grad(ctx.emb_shape, lists, sites)
        return (None, dsrc, None, demb, None) + tuple(grads_w)


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


class _PoolAggregateRowsFn(torch.autograd.Function):
    """y = agg.aggregate_rows(src, segments) for MaxPoolingAggregator / MeanPoolingAggregator on the unfused fp32 path
    (gather -> Dense(relu, bias) -> pool over the fanout -> both matmuls), differentiable w.r.t. the four weight tensors
    and (layers >= 1) src, and (layer 0, identity_dim > 0) `emb`, the [N+1, d] embedding view of src's first d columns.
    The gathered neighbour rows and the MLP activations are kept for the backward pass."""

    @staticmethod
    def forward(ctx, agg, src, segments, Ws, Wn, Wm, bm, emb=None, sites=None):
        """sites: None, or one (seed, call, rate) per segment for the MLP input (training dropout, layers.py:107; the self
        rows are not dropped); the kept xn is the dropped input, which is what dWm = xn^T dpre needs."""
        code, post = act_code(agg.act)
        if post is not None:
            raise NotImplementedError("training supports act=relu or identity")
        if len(agg.mlp_layers) != 1 or agg.dropout:
            raise NotImplementedError("training supports one MLP layer and dropout = 0")
        F_in, hid = src.shape[1], agg.hidden_dim
        rows = max(s.out_row0 + s.n for s in segments)
        with torch.no_grad():
            xs = torch.empty((rows, ops.pad_cols(F_in)), dtype=torch.float32, device=src.device)[:, :F_in]
            hp = torch.empty((rows, hid), dtype=torch.float32, device=src.device)
            kept = []
            for si, s in enumerate(segments):
                n, k = s.n, s.k
                xn = ops.gather_rows(src, s.neigh_ids[:n * k]) if s.neigh_ids is not None else \
                    src[s.neigh_row0:s.neigh_row0 + n * k]
                if sites is not None:                        # out of place: layer >= 1 rows belong to the previous layer
                    xn = ops.dropout_apply(xn, sites[si])
                mlp = agg.mlp_layers[0]
                mlp.math = agg.math
                h = mlp(xn)
                if agg.pool == "mean":
                    hp[s.out_row0:s.out_row0 + n] = ops.gather_mean(h, [ops.Seg(n, k)], want_self=False, out_pitch=hid)[1]
                else:
                    hp[s.out_row0:s.out_row0 + n] = ops.segment_max(h, n, k)
                if s.self_ids is not None:
                    ops.gather_rows(src, s.self_ids[:n], out=xs[s.out_row0:s.out_row0 + n])
                else:
                    xs[s.out_row0:s.out_row0 + n] = src[s.self_row0:s.self_row0 + n]
                kept.extend([xn, h])
            y = agg._finish([(xs, agg.input_dim, Ws), (hp, hid, Wn)], agg._combine())
        ctx.pool, ctx.relu, ctx.concat = agg.pool, code == ops.ACT_RELU, bool(agg.concat)
        ctx.segments, ctx.src_shape, ctx.F_in, ctx.sites = segments, tuple(src.shape), F_in, sites
        ctx.src_needs_grad = bool(torch.is_tensor(src) and src.requires_grad)
        ctx.emb_shape = tuple(emb.shape) if emb is not None and emb.requires_grad else None
        ctx.save_for_backward(xs, hp, y, Ws, Wn, Wm, *kept)
        return y

    @staticmethod
    def backward(ctx, dy):
        xs, hp, y, Ws, Wn, Wm = ctx.saved_tensors[:6]
        kept = ctx.saved_tensors[6:]
        F_in = ctx.F_in
        dz = dy * (y > 0).to(dy.dtype) if ctx.relu else dy
        D = Ws.shape[1]
        dz_s, dz_n = (dz[:, :D], dz[:, D:]) if ctx.concat else (dz, dz)
        dWs, dWn = xs.t() @ dz_s, hp.t() @ dz_n
        dhp = dz_n @ Wn.t()
        dWm, dbm = torch.zeros_like(Wm), torch.zeros(Wm.shape[1], dtype=dy.dtype, device=dy.device)
        dsrc = torch.zeros(ctx.src_shape, dtype=dy.dtype, device=dy.device) if ctx.src_needs_grad else None
        dxs = dz_s @ Ws.t() if ctx.src_needs_grad else None
        emb = ctx.emb_shape is not None
        d = ctx.emb_shape[1] if emb else 0
        # the embedding columns only need dZ @ W[:d]^T (feature columns are not trainable)
        es = dz_s @ Ws[:d].t() if emb else None
        W_dx = Wm if ctx.src_needs_grad else Wm[:d]
        lists = []
        for i, s in enumerate(ctx.segments):
            n, k = s.n, s.k
            rows = slice(s.out_row0, s.out_row0 + n)
            xn, h = kept[2 * i][:, :F_in], kept[2 * i + 1]
            g_wm, g_bm, dxn = pool_branch_backward(ctx.pool, xn, h, hp[rows], dhp[rows], W_dx, k,
                                                   ctx.src_needs_grad or emb)
            dWm += g_wm
            dbm += g_bm
            if dxn is not None and ctx.sites is not None:    # through the input mask, regenerated
                dxn = ops.dropout_apply(dxn, ctx.sites[i])
            if emb:                                          # self id: dxs; neighbour id of gathered row r: dxn[r]
                lists += [(s.self_ids[:n], es[rows], 1, 1.0), (s.neigh_ids[:n * k], dxn[:, :d], 1, 1.0)]
            if ctx.src_needs_grad:
                if s.self_ids is not None or s.neigh_ids is not None:
                    raise NotImplementedError("gradient w.r.t. an id-addressed source (trainable features) is out of scope")
                dsrc[s.neigh_row0:s.neigh_row0 + n * k] += dxn
                dsrc[s.self_row0:s.self_row0 + n] += dxs[rows]
        demb = _embedding_grad(ctx.emb_shape, lists) if emb else None
        return None, dsrc, None, dWs, dWn, dWm, dbm, demb, None


class _SeqAggregateRowsFn(torch.autograd.Function):
    """y = agg.aggregate_rows(src, segments) for SeqAggregator, differentiable w.r.t. Ws, Wn, the cell's kernel and bias,
    (layers >= 1) src and (layer 0, identity_dim > 0) `emb`, the [N+1, d] embedding view of src's first d columns.
    Forward per hop: X (gathered rows, or the previous layer's row range) -> lengths (gs_seq_lengths) -> P = X W_x + b
    (library GEMM, agg.math) -> gs_lstm_forward, keeping X, the lengths, the gates, c and h_{t-1}.  Backward per hop:
    gs_lstm_backward gives dZ; dW_x = X^T dZ, dW_h = h_prev^T dZ, db = sum dZ and dX = dZ W_x^T are library matmuls."""

    @staticmethod
    def forward(ctx, agg, src, segments, Ws, Wn, kernel, cell_bias, emb=None):
        code, post = act_code(agg.act)
        if post is not None:
            raise NotImplementedError("training supports act=relu or identity")
        refuse_seq_table(src)
        F_in, H = src.shape[1], agg.hidden_dim
        rows = max(s.out_row0 + s.n for s in segments)
        with torch.no_grad():
            xs = torch.empty((rows, ops.pad_cols(F_in)), dtype=torch.float32, device=src.device)[:, :F_in]
            hl = torch.empty((rows, H), dtype=torch.float32, device=src.device)
            Wx, Wh = kernel[:F_in], kernel[F_in:]
            kept = []
            for s in segments:
                n, k = s.n, s.k
                X = ops.gather_rows(src, s.neigh_ids[:n * k]) if s.neigh_ids is not None else \
                    src[s.neigh_row0:s.neigh_row0 + n * k]
                lengths = ops.seq_lengths(X, n, k)
                P = ops.sage_gemm([(X, F_in, Wx)], bias=cell_bias, math=agg.math)
                _, gates, c, h_prev = ops.lstm_forward(P, Wh, lengths, n, k, out=hl[s.out_row0:s.out_row0 + n], train=True)
                del P
                if s.self_ids is not None:
                    ops.gather_rows(src, s.self_ids[:n], out=xs[s.out_row0:s.out_row0 + n])
                else:
                    xs[s.out_row0:s.out_row0 + n] = src[s.self_row0:s.self_row0 + n]
                kept.extend([X, lengths, gates, c, h_prev])
            y = agg._finish([(xs, agg.input_dim, Ws), (hl, H, Wn)], agg._combine())
        ctx.relu, ctx.concat = code == ops.ACT_RELU, bool(agg.concat)
        ctx.segments, ctx.src_shape, ctx.F_in = segments, tuple(src.shape), F_in
        ctx.src_needs_grad = bool(torch.is_tensor(src) and src.requires_grad)
        ctx.emb_shape = tuple(emb.shape) if emb is not None and emb.requires_grad else None
        ctx.save_for_backward(xs, hl, y, Ws, Wn, kernel, *kept)
        return y

    @staticmethod
    def backward(ctx, dy):
        xs, hl, y, Ws, Wn, kernel = ctx.saved_tensors[:6]
        kept = ctx.saved_tensors[6:]
        F_in = ctx.F_in
        dz = dy * (y > 0).to(dy.dtype) if ctx.relu else dy
        D = Ws.shape[1]
        dz_s, dz_n = (dz[:, :D], dz[:, D:]) if ctx.concat else (dz, dz)
        dWs, dWn = xs.t() @ dz_s, hl.t() @ dz_n
        dhl = (dz_n @ Wn.t()).contiguous()
        Wx, Wh = kernel[:F_in], kernel[F_in:]
        dWx, dWh = torch.zeros_like(Wx), torch.zeros_like(Wh)
        db = torch.zeros(kernel.shape[1], dtype=dy.dtype, device=dy.device)
        dsrc = torch.zeros(ctx.src_shape, dtype=dy.dtype, device=dy.device) if ctx.src_needs_grad else None
        dxs = dz_s @ Ws.t() if ctx.src_needs_grad else None
        emb = ctx.emb_shape is not None
        d = ctx.emb_shape[1] if emb else 0
        es = dz_s @ Ws[:d].t() if emb else None          # the embedding columns only need dZ @ W[:d]^T
        lists = []
        for i, s in enumerate(ctx.segments):
            n, k = s.n, s.k
            rows = slice(s.out_row0, s.out_row0 + n)
            X, lengths, gates, c, h_prev = kept[5 * i:5 * i + 5]
            dZ = ops.lstm_backward(dhl[rows], gates, c, lengths, Wh, n, k)
            dWx += X.t() @ dZ
            dWh += h_prev.t() @ dZ
            db += dZ.sum(dim=0)
            if emb:                                      # self id: dxs; neighbour id of gathered row r: dX[r]
                lists += [(s.self_ids[:n], es[rows], 1, 1.0), (s.neigh_ids[:n * k], dZ @ Wx[:d].t(), 1, 1.0)]
            if ctx.src_needs_grad:
                if s.self_ids is not None or s.neigh_ids is not None:
                    raise NotImplementedError("gradient w.r.t. an id-addressed source (trainable features) is out of scope")
                dsrc[s.neigh_row0:s.neigh_row0 + n * k] += dZ @ Wx.t()
                dsrc[s.self_row0:s.self_row0 + n] += dxs[rows]
        demb = _embedding_grad(ctx.emb_shape, lists) if emb else None
        return None, dsrc, None, dWs, dWn, torch.cat([dWx, dWh]), db, demb


FUSED_POOL_MAX_FANOUT, FUSED_POOL_MAX_K = 128, 640       # K4's limits (include/graphsage_b200.h)


def refuse_fused_pool(model):
    """The limits of the fused bf16 pooling branch (fused_pool=True) that are known once the aggregators exist."""
    if not getattr(model, "fused_pool", False):
        return
    if not hasattr(model.aggregators[0], "mlp_layers"):
        raise NotImplementedError("fused_pool=True applies to the maxpool and meanpool aggregators only")
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
        if agg.hidden_dim % 128 != 0:
            raise NotImplementedError("fused_pool=True needs a pooling hidden width that is a multiple of 128 (got %d)"
                                      % agg.hidden_dim)
        if len(agg.mlp_layers) != 1:
            raise NotImplementedError("fused_pool=True supports one MLP layer")


class _FusedPoolAggregateRowsFn(torch.autograd.Function):
    """y = agg.aggregate_rows(src, segments) for MaxPoolingAggregator / MeanPoolingAggregator through the fused bf16
    kernels (fused_pool=True): the pooled branch is K4 (ops.maxpool_mlp_fused) in the forward; the backward recomputes
    the MLP tile instead of storing it (B1 ops.pool_mlp_backward_dp), then dWm / dbm (B2) and, where a source gradient
    is needed, dX (B3).  bf16 operands with fp32 accumulation whatever agg.math is; the self branch and the Ws / Wn
    gradients are those of _PoolAggregateRowsFn.  Saved: the self rows, the pooled rows, y, the weights and the bf16
    operand table - neither the gathered neighbour rows nor the MLP activations."""

    @staticmethod
    def forward(ctx, agg, src, segments, Ws, Wn, Wm, bm, emb=None, persistent=False):
        """persistent: src is the model's feature table (layer 0), cast to bf16 once per table version; a layer >= 1
        source is cast on every call and the cast is kept for the backward."""
        code, post = act_code(agg.act)
        if post is not None:
            raise NotImplementedError("training supports act=relu or identity")
        if hasattr(src, "c_table"):
            raise NotImplementedError("fused_pool=True with a node-partitioned (ShardedFeatures) table is not implemented")
        F_in, hid = src.shape[1], agg.hidden_dim
        for s in segments:
            if s.k > FUSED_POOL_MAX_FANOUT or F_in > FUSED_POOL_MAX_K or hid % 128 != 0:
                raise NotImplementedError("fused_pool=True needs fanout <= %d, input width <= %d and hidden %% 128 == 0 "
                                          "(k=%d K=%d hidden=%d)" % (FUSED_POOL_MAX_FANOUT, FUSED_POOL_MAX_K, s.k, F_in, hid))
        rows = max(s.out_row0 + s.n for s in segments)
        with torch.no_grad():
            table = agg._bf16_table(src, persistent)
            if getattr(agg, "_packed_mlp", None) is None:
                agg._packed_mlp = ops.PackedMlpWeights()
            hp = torch.empty((rows, hid), dtype=torch.float32, device=src.device)
            xs = torch.empty((rows, ops.pad_cols(F_in)), dtype=torch.float32, device=src.device)[:, :F_in]
            for s in segments:
                ops.maxpool_mlp_fused(table, s.n, s.k, Wm, bm, agg._packed_mlp, row_ids=s.neigh_ids, row0=s.neigh_row0,
                                      K=F_in, out=hp[s.out_row0:s.out_row0 + s.n], pool=agg.pool)
                ops.gather_rows_f32(src, ids=None if s.self_ids is None else s.self_ids[:s.n], row0=s.self_row0, n=s.n,
                                    out=xs[s.out_row0:s.out_row0 + s.n])
            y = agg._finish([(xs, agg.input_dim, Ws), (hp, hid, Wn)], agg._combine())
        ctx.agg, ctx.relu, ctx.concat = agg, code == ops.ACT_RELU, bool(agg.concat)
        ctx.segments, ctx.src_shape, ctx.F_in = segments, tuple(src.shape), F_in
        ctx.src_needs_grad = bool(torch.is_tensor(src) and src.requires_grad)
        ctx.emb_shape = tuple(emb.shape) if emb is not None and emb.requires_grad else None
        ctx.save_for_backward(xs, hp, y, Ws, Wn, Wm, bm, table)
        return y

    @staticmethod
    def backward(ctx, dy):
        xs, hp, y, Ws, Wn, Wm, bm, table = ctx.saved_tensors
        agg, F_in = ctx.agg, ctx.F_in
        dz = dy * (y > 0).to(dy.dtype) if ctx.relu else dy
        D = Ws.shape[1]
        dz_s, dz_n = (dz[:, :D], dz[:, D:]) if ctx.concat else (dz, dz)
        dWs, dWn = xs.t() @ dz_s, hp.t() @ dz_n
        dhp = (dz_n @ Wn.t()).contiguous()
        dWm, dbm = torch.zeros_like(Wm), torch.zeros(Wm.shape[1], dtype=dy.dtype, device=dy.device)
        dsrc = torch.zeros(ctx.src_shape, dtype=dy.dtype, device=dy.device) if ctx.src_needs_grad else None
        dxs = dz_s @ Ws.t() if ctx.src_needs_grad else None
        emb = ctx.emb_shape is not None
        d = ctx.emb_shape[1] if emb else 0
        es = dz_s @ Ws[:d].t() if emb else None
        packed_dx = None
        if ctx.src_needs_grad or emb:                        # dX columns: all of them for a previous layer, else [0, d)
            cols = F_in if ctx.src_needs_grad else d
            if getattr(agg, "_packed_dx", None) is None or agg._packed_dx.cols != cols:
                agg._packed_dx = ops.PackedMlpDxWeights(cols)
            packed_dx = agg._packed_dx
        lists = []
        for s in ctx.segments:                               # per hop, in order: B1 -> B2 (dWm, dbm) -> B3
            n, k = s.n, s.k
            rows = slice(s.out_row0, s.out_row0 + n)
            grad = ops.pool_mlp_backward_dp(table, n, k, Wm, bm, agg._packed_mlp, dhp[rows], row_ids=s.neigh_ids,
                                            row0=s.neigh_row0, K=F_in, pool=agg.pool)
            ops.pool_mlp_backward_dw(table, n, k, grad, dWm, dbm, row_ids=s.neigh_ids, row0=s.neigh_row0, K=F_in)
            if packed_dx is None:
                continue
            dxn = ops.pool_mlp_backward_dx(grad, n, k, Wm, packed_dx)
            if emb:                                          # self id: dxs; neighbour id of gathered row r: dxn[r]
                lists += [(s.self_ids[:n], es[rows], 1, 1.0), (s.neigh_ids[:n * k], dxn[:, :d], 1, 1.0)]
            if ctx.src_needs_grad:
                if s.self_ids is not None or s.neigh_ids is not None:
                    raise NotImplementedError("gradient w.r.t. an id-addressed source (trainable features) is out of scope")
                dsrc[s.neigh_row0:s.neigh_row0 + n * k] += dxn
                dsrc[s.self_row0:s.self_row0 + n] += dxs[rows]
        demb = _embedding_grad(ctx.emb_shape, lists) if emb else None
        return None, dsrc, None, dWs, dWn, dWm, dbm, demb, None


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
    src = model.features
    pool = hasattr(model.aggregators[0], "mlp_layers")
    seq = hasattr(model.aggregators[0], "cell")
    plan = dropout_site_plan("seq" if seq else "maxpool" if pool else "mean", L) if dropout else []
    call = {site: model.dropout_counter + i for i, site in enumerate(plan)}
    for layer in range(L):
        hops = L - layer
        row0 = [sum(counts[:h]) for h in range(hops + 1)]
        segs = []
        for hop in range(hops):
            k = num_samples[L - hop - 1]
            if layer == 0:
                segs.append(ops.Seg(counts[hop], k, self_ids=samples[hop], neigh_ids=samples[hop + 1],
                                    out_row0=row0[hop]))
            else:
                segs.append(ops.Seg(counts[hop], k, self_row0=row0[hop], neigh_row0=row0[hop + 1],
                                    out_row0=row0[hop]))
        agg = model.aggregators[layer]
        # layer 0 reads the embedding table (identity_dim > 0) through src; handing it over as an input lets autograd
        # deliver the scattered gradient as embeds.grad
        emb = getattr(model, "embeds", None) if layer == 0 else None
        sites = None
        if dropout and not seq:                              # per hop: the MLP-input site, or the (neighbour, self) pair
            key, dev = model.dropout_key, model.dropout_call_dev
            if pool:
                sites = [(key, call[(layer, h, "mlp")], dropout, dev) for h in range(hops)]
            else:
                sites = [((key, call[(layer, h, "neigh")], dropout, dev), (key, call[(layer, h, "self")], dropout, dev))
                         for h in range(hops)]
        if seq:                                              # LSTM: draws no dropout mask
            cell = agg.cell.vars
            src = _SeqAggregateRowsFn.apply(agg, src, segs, agg.vars["self_weights"], agg.vars["neigh_weights"],
                                            cell["kernel"], cell["bias"], emb)
        elif pool and fused:                                 # max-pool / mean-pool through the bf16 kernels
            mlp = agg.mlp_layers[0].vars
            src = _FusedPoolAggregateRowsFn.apply(agg, src, segs, agg.vars["self_weights"], agg.vars["neigh_weights"],
                                                  mlp["weights"], mlp["bias"], emb, layer == 0)
        elif pool:                                           # max-pool / mean-pool
            mlp = agg.mlp_layers[0].vars
            src = _PoolAggregateRowsFn.apply(agg, src, segs, agg.vars["self_weights"], agg.vars["neigh_weights"],
                                             mlp["weights"], mlp["bias"], emb, sites)
        else:
            ws = (agg.vars["weights"],) if "weights" in agg.vars else (agg.vars["self_weights"], agg.vars["neigh_weights"])
            src = _AggregateRowsFn.apply(agg, src, segs, emb, sites, *ws)
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
        super(SupervisedGraphsage, self).__init__(placeholders, features, adj, degrees, layer_infos, concat=concat,
                                                  aggregator_type=aggregator_type, model_size=model_size,
                                                  identity_dim=identity_dim, device=device, **kwargs)
        if aggregator_type not in ("mean", "gcn", "maxpool", "meanpool", "seq"):
            raise NotImplementedError("training is implemented for the mean, gcn, maxpool, meanpool and seq aggregators")
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
        return out @ self.node_pred_vars["weights"] + self.node_pred_vars["bias"]

    def loss(self, batch, labels, dropout=0.):
        """supervised_models.py:101-118: weight decay * l2_loss(var) over aggregator + head variables, then the
        mean of the per-element sigmoid xent (multi-label) or the mean of the per-node softmax xent."""
        logits = self.logits(batch, dropout=dropout) if dropout else self.logits(batch)    # overrides take (batch)
        labels = labels.to(device=logits.device, dtype=torch.float32)
        loss = classification_loss(logits, labels, self.sigmoid_loss)
        if self.weight_decay:
            loss = loss + weight_decay_term(self.decayed_parameters(), self.weight_decay)
        return loss

    def train_step(self, batch, labels):
        """One Adam step at the training dropout rate placeholders['dropout'] (supervised_train.py:271)."""
        self.optimizer.zero_grad(set_to_none=True)
        loss = self.loss(batch, labels, dropout=self.dropout_rate)
        loss.backward()
        if self.distributed:                                                     # data parallel: mean gradient over ranks
            from .parallel import allreduce_gradients
            self.last_allreduce_bytes = allreduce_gradients(self.parameters(), self.group)
        for p in self.parameters():                                              # clip_by_value(grad, -5, 5)  :93-94
            if p.grad is not None:
                p.grad.clamp_(-5.0, 5.0)
        self.optimizer.step()
        return loss.detach()

    def graphed_train_step(self, batch_size):
        """train_step for a fixed batch size captured in one CUDA graph: returns step(batch, labels) -> loss, a static 0-d
        CUDA tensor (see graphed_training.GraphedTrainStep; a short last batch runs through the eager train_step)."""
        return GraphedTrainStep(self, batch_size)

    def predict(self, batch):
        with torch.no_grad():
            lg = self.logits(batch)
            return torch.sigmoid(lg) if self.sigmoid_loss else torch.softmax(lg, dim=1)
