"""MeanAggregator / GCNAggregator / MaxPoolingAggregator / MeanPoolingAggregator / TwoMaxLayerPoolingAggregator /
SeqAggregator - the surface of
reference graphsage/aggregators.py over the library's CUDA kernels.

Two entry points per aggregator:
  agg((self_vecs[n, in], neigh_vecs[n, k, neigh_in])) -> [n, out * (2 if concat else 1)]
      the reference call convention (dense, already-gathered inputs);
  agg.aggregate_rows(src, segments) -> [rows, out_w]
      the gather-fused form used by SampleAndAggregate.aggregate: neighbours are addressed by
      id lists (or row ranges) into `src`, the [n*k, F] neighbour tensor is never materialised.
"""
import torch

from . import ops
from .inits import glorot, zeros
from .layers import Dense, Layer, act_code, identity, relu  # noqa: F401  (relu/identity re-exported as `act` values)

_DEFAULT_MATH = [ops.MATH_FP32_SIMT]
_MATH_NAMES = {"fp32": ops.MATH_FP32_SIMT, "simt": ops.MATH_FP32_SIMT, "tf32x3": ops.MATH_TF32X3,
               "tf32": ops.MATH_TF32, "bf16": ops.MATH_BF16}


def set_default_math(mode):
    """Arithmetic of the dense contraction for aggregators created afterwards: 'fp32' (CUDA cores),
    'tf32x3' (tensor cores, fp32-accurate), 'tf32', 'bf16'."""
    _DEFAULT_MATH[0] = _MATH_NAMES[mode] if isinstance(mode, str) else int(mode)


def _dropout(x, p):
    return torch.nn.functional.dropout(x, p=float(p), training=True) if p else x


def _dense_segment(n, k):
    return [ops.make_segment(n, k)]


def _rows(src, ids, row0, n, f32=False, out=None):
    """Rows ids[:n] (or row0 .. row0 + n) of src: gathered by the library (gs_gather_rows_f32, which widens a bf16 table,
    when f32 is set), or else a view of the row range (copied into `out` when given)."""
    if f32:
        return ops.gather_rows_f32(src, ids=None if ids is None else ids[:n], row0=row0, n=n, out=out)
    if ids is not None:
        return ops.gather_rows(src, ids[:n], out=out)
    if out is None:
        return src[row0:row0 + n]
    out.copy_(src[row0:row0 + n])
    return out


# K4's limits (include/graphsage_b200.h): fanout, layer input width, multiple of the pooling hidden width
FUSED_POOL_MAX_FANOUT, FUSED_POOL_MAX_K, FUSED_POOL_HIDDEN_STEP = 128, 640, 128


def fused_pool_fits(k, K, hidden):
    return k <= FUSED_POOL_MAX_FANOUT and K <= FUSED_POOL_MAX_K and hidden % FUSED_POOL_HIDDEN_STEP == 0


# K5's limits: as K4's, and the second layer's width a multiple of 256 (one CTA's slice of it)
FUSED_POOL2_H2_STEP = 256


def fused_pool2_fits(k, K, h1, h2):
    return fused_pool_fits(k, K, h1) and h2 % FUSED_POOL2_H2_STEP == 0


class _SageAggregator(Layer):
    def _combine(self):
        return ops.COMBINE_CONCAT if self.concat and "self_weights" in self.vars else ops.COMBINE_ADD

    def _summarise(self, src, segments, hop, f32_self=False):
        """The GEMM parts [self rows, neighbour summary] of a layer whose neighbour branch is a per-hop summary of
        hidden_dim columns (pools, seq): hop(i, s, out) writes the summary of segment i (s) into `out`, its rows of the
        summary part; each hop's self rows are copied after it."""
        rows = max(s.out_row0 + s.n for s in segments)
        F_in = src.shape[1]
        xs = torch.empty((rows, ops.pad_cols(F_in)), dtype=torch.float32, device=src.device)[:, :F_in]
        h = torch.empty((rows, self.hidden_dim), dtype=torch.float32, device=src.device)
        for i, s in enumerate(segments):
            hop(i, s, h[s.out_row0:s.out_row0 + s.n])
            _rows(src, s.self_ids, s.self_row0, s.n, f32_self, out=xs[s.out_row0:s.out_row0 + s.n])
        return [(xs, self.input_dim, self.vars["self_weights"]), (h, self.hidden_dim, self.vars["neigh_weights"])]

    def _finish(self, parts, combine):
        code, post = act_code(self.act)
        if getattr(self, "_packed", None) is None:
            self._packed = ops.PackedWeights()
        y = ops.sage_gemm(parts, combine=combine, bias=self.vars.get("bias"), act=code, math=self.math,
                          packed=self._packed)
        return post(y) if post else y

    def _small_layer(self, src, segments, parts, combine, include_self, final):
        """Whole layer in one launch when it is small (last layers: B rows).  Returns None if not applicable."""
        code, post = act_code(self.act)
        if (len(segments) != 1 or not torch.is_tensor(src) or post is not None or self.dropout
                or segments[0].out_row0 + segments[0].n > ops.SMALL_LAYER_MAX_ROWS or src.shape[1] > 2048
                or any(K != src.shape[1] for (_, K, _) in parts)
                or (sum(B.shape[1] for (_, _, B) in parts) if combine == ops.COMBINE_CONCAT else parts[0][2].shape[1]) > 1024):
            return None       # gs_sage_layer_small limits: rows, K <= 2048, total output width <= 1024
        l2 = bool(final and final.get("l2_normalize"))
        bump = final.get("bump") if final else None
        y = ops.sage_layer_small(src, segments[0], parts, combine=combine, include_self=include_self,
                                 bias=self.vars.get("bias"), act=code, l2_normalize=l2,
                                 counter_dev=None if bump is None else bump[0], counter_inc=0 if bump is None else bump[1])
        if final is not None:
            final["normalized"] = l2
            final["bumped"] = bump is not None
        return y

    @property
    def output_width(self):
        return self.output_dim * (2 if (self.concat and "self_weights" in self.vars) else 1)


class MeanAggregator(_SageAggregator):
    """act(concat_or_add(self @ self_weights, mean_k(neigh) @ neigh_weights)) - aggregators.py:43-64."""

    def __init__(self, input_dim, output_dim, neigh_input_dim=None, dropout=0., bias=False, act=relu, name=None,
                 concat=False, device="cuda", **kwargs):
        super(MeanAggregator, self).__init__(**kwargs)
        self.dropout = dropout
        self.bias = bias
        self.act = act
        self.concat = concat
        if neigh_input_dim is None:
            neigh_input_dim = input_dim
        self.vars["neigh_weights"] = glorot([neigh_input_dim, output_dim], name="neigh_weights", device=device)
        self.vars["self_weights"] = glorot([input_dim, output_dim], name="self_weights", device=device)
        if self.bias:   # the reference dereferences self.output_dim too early here (aggregators.py:34-35); fixed, not replicated
            self.vars["bias"] = zeros([output_dim * (2 if concat else 1)], name="bias", device=device)
        self.input_dim = input_dim
        self.output_dim = output_dim
        self.neigh_input_dim = neigh_input_dim
        self.math = _DEFAULT_MATH[0]

    def _call(self, inputs):
        self_vecs, neigh_vecs = inputs
        n, k, d = neigh_vecs.shape
        neigh_vecs = _dropout(neigh_vecs, self.dropout)
        self_vecs = _dropout(self_vecs, self.dropout)
        _, means = ops.gather_mean(neigh_vecs.reshape(n * k, d), _dense_segment(n, k), want_self=False)
        return self._finish([(self_vecs, self.input_dim, self.vars["self_weights"]),
                             (means, self.neigh_input_dim, self.vars["neigh_weights"])], self._combine())

    def aggregate_rows(self, src, segments, final=None, src_persistent=False):
        if self.dropout:
            raise NotImplementedError("dropout > 0 uses the dense call path")
        y = self._small_layer(src, segments, [(None, self.input_dim, self.vars["self_weights"]),
                                              (None, self.neigh_input_dim, self.vars["neigh_weights"])],
                              self._combine(), False, final)
        if y is not None:
            return y
        if torch.is_tensor(src) and src.is_cuda and src.dtype == torch.float32 and all(s.self_ids is not None for s in segments):
            # the self rows only feed the GEMM: it reads them from the table by id, so the gather neither fetches them nor
            # writes a copy (same operand values, same bits)
            _, xm = ops.gather_mean(src, segments, want_self=False)
            xs = ops.TableRows(src, [(s.self_ids[:s.n], s.out_row0) for s in segments], xm.shape[0])
        else:
            xs, xm = ops.gather_mean(src, segments, want_self=True)
        return self._finish([(xs, self.input_dim, self.vars["self_weights"]),
                             (xm, self.neigh_input_dim, self.vars["neigh_weights"])], self._combine())


class GCNAggregator(_SageAggregator):
    """act(mean_{k+1}(neigh U self) @ weights) - aggregators.py:101-116 (single weight, concat ignored)."""

    def __init__(self, input_dim, output_dim, neigh_input_dim=None, dropout=0., bias=False, act=relu, name=None,
                 concat=False, device="cuda", **kwargs):
        super(GCNAggregator, self).__init__(**kwargs)
        self.dropout = dropout
        self.bias = bias
        self.act = act
        self.concat = concat
        if neigh_input_dim is None:
            neigh_input_dim = input_dim
        self.vars["weights"] = glorot([neigh_input_dim, output_dim], name="neigh_weights", device=device)
        if self.bias:
            self.vars["bias"] = zeros([output_dim], name="bias", device=device)
        self.input_dim = input_dim
        self.output_dim = output_dim
        self.neigh_input_dim = neigh_input_dim
        self.math = _DEFAULT_MATH[0]

    def _call(self, inputs):
        self_vecs, neigh_vecs = inputs
        n, k, d = neigh_vecs.shape
        if self_vecs.shape[1] != d:
            raise ValueError("GCNAggregator needs self and neighbour vectors of equal width")
        neigh_vecs = _dropout(neigh_vecs, self.dropout)
        self_vecs = _dropout(self_vecs, self.dropout)
        # one source matrix: neighbours first, then the self rows
        src = torch.cat([neigh_vecs.reshape(n * k, d), self_vecs], dim=0)
        seg = [ops.make_segment(n, k, self_row0=n * k, neigh_row0=0)]
        _, means = ops.gather_mean(src, seg, include_self=True, want_self=False)
        return self._finish([(means, self.neigh_input_dim, self.vars["weights"])], ops.COMBINE_ADD)

    def aggregate_rows(self, src, segments, final=None, src_persistent=False):
        if self.dropout:
            raise NotImplementedError("dropout > 0 uses the dense call path")
        y = self._small_layer(src, segments, [(None, self.neigh_input_dim, self.vars["weights"])], ops.COMBINE_ADD, True,
                              final)
        if y is not None:
            return y
        _, means = ops.gather_mean(src, segments, include_self=True, want_self=False)
        return self._finish([(means, self.neigh_input_dim, self.vars["weights"])], ops.COMBINE_ADD)


class MaxPoolingAggregator(_SageAggregator):
    """act(concat_or_add(self @ Ws, max_k(relu(neigh @ Wm + bm)) @ Wn)) - aggregators.py:119-195,
    with Dense (layers.py:73-116) as the single MLP layer; hidden 512 ("small") / 1024 ("big")."""

    def __init__(self, input_dim, output_dim, model_size="small", neigh_input_dim=None, dropout=0., bias=False,
                 act=relu, name=None, concat=False, device="cuda", **kwargs):
        super(MaxPoolingAggregator, self).__init__(**kwargs)
        self.dropout = dropout
        self.bias = bias
        self.act = act
        self.concat = concat
        if neigh_input_dim is None:
            neigh_input_dim = input_dim
        if model_size == "small":
            hidden_dim = self.hidden_dim = 512
        elif model_size == "big":
            hidden_dim = self.hidden_dim = 1024
        else:
            raise ValueError("model_size must be 'small' or 'big'")
        self.math = _DEFAULT_MATH[0]
        self.mlp_layers = [Dense(input_dim=neigh_input_dim, output_dim=hidden_dim, act=relu, dropout=dropout,
                                 sparse_inputs=False, logging=self.logging, device=device, math=self.math)]
        self.vars["neigh_weights"] = glorot([hidden_dim, output_dim], name="neigh_weights", device=device)
        self.vars["self_weights"] = glorot([input_dim, output_dim], name="self_weights", device=device)
        if self.bias:
            self.vars["bias"] = zeros([output_dim * (2 if concat else 1)], name="bias", device=device)
        self.input_dim = input_dim
        self.output_dim = output_dim
        self.neigh_input_dim = neigh_input_dim

    pool = "max"

    def _mlp(self, rows):
        h = rows
        for layer in self.mlp_layers:
            layer.math = self.math
            h = layer(h)
        return h

    def _pool(self, h, n, k):
        if self.pool == "mean":
            return ops.gather_mean(h, [ops.Seg(n, k)], want_self=False, out_pitch=h.shape[1])[1]
        return ops.segment_max(h, n, k)

    def _call(self, inputs):
        self_vecs, neigh_vecs = inputs
        n, k, d = neigh_vecs.shape
        hmax = self._pool(self._mlp(neigh_vecs.reshape(n * k, d)), n, k)
        return self._finish([(self_vecs, self.input_dim, self.vars["self_weights"]),
                             (hmax, self.hidden_dim, self.vars["neigh_weights"])], self._combine())

    def _bf16_table(self, src, persistent):
        """K4's operand table: bf16 rows with a 16-byte-multiple pitch.  A bf16 source is used as is.  An fp32 source is
        cast by gs_cast_rows_bf16 - once per tensor version when the caller says it is the persistent feature table
        (layer 0), on EVERY call otherwise: intermediate activations are fresh torch.empty buffers the C library
        fills, so neither their address nor their _version tells one step's values from the next."""
        if src.dtype == torch.bfloat16:
            if src.stride(0) % 8 != 0 or src.data_ptr() % 16 != 0:
                raise ValueError("bfloat16 source rows must be 16-byte aligned multiples (pitch % 8 == 0)")
            return src
        if not persistent or ops.REPACK_ALWAYS[0]:
            return ops.cast_rows_bf16(src)
        key = (ops.CACHE_EPOCH[0], src.data_ptr(), src._version, tuple(src.shape))
        if getattr(self, "_bf16_ref", None) is not src or getattr(self, "_bf16_key", None) != key:
            self._bf16_src, self._bf16_ref, self._bf16_key = ops.cast_rows_bf16(src), src, key
        return self._bf16_src

    def _fused_ok(self, src, segments):
        return (self.math == ops.MATH_BF16 and torch.is_tensor(src) and not self.dropout and len(self.mlp_layers) == 1
                and all(fused_pool_fits(s.k, self.neigh_input_dim, self.hidden_dim) for s in segments)
                and self.mlp_layers[0].act is relu and "bias" in self.mlp_layers[0].vars)

    def _fused_hop(self, table, s, out):
        """K4 for one hop: gather -> MLP -> ReLU -> pool over the fanout in one wgmma kernel (bf16 operands) into `out`."""
        if getattr(self, "_packed_mlp", None) is None:
            self._packed_mlp = ops.PackedMlpWeights()
        mlp = self.mlp_layers[0].vars
        ops.maxpool_mlp_fused(table, s.n, s.k, mlp["weights"], mlp["bias"], self._packed_mlp, row_ids=s.neigh_ids,
                              row0=s.neigh_row0, K=self.neigh_input_dim, out=out, pool=self.pool)

    def _pooled_parts(self, src, segments, kept=None, sites=None):
        """The GEMM parts of the materialised form: per hop the neighbour rows (widened to fp32 from a bf16 table), then
        the MLP and the pooling kernel.  With training dropout each Dense layer's input is masked first: sites[hop] is
        the one site of a one-layer MLP, the (mlp, mlp2) pair of a two-layer one.  `kept` (training) receives each hop's
        Dense inputs (as masked) and the last Dense's output."""
        widen = torch.is_tensor(src) and src.dtype != torch.float32

        def hop(i, s, out):
            h = _rows(src, s.neigh_ids, s.neigh_row0, s.n * s.k, widen)
            hop_sites = None if sites is None else (sites[i],) if len(self.mlp_layers) == 1 else sites[i]
            for j, layer in enumerate(self.mlp_layers):
                if hop_sites is not None:           # out of place: layer >= 1 rows belong to the previous layer
                    h = ops.dropout_apply(h, hop_sites[j])
                if kept is not None:
                    kept.append(h)
                layer.math = self.math
                h = layer(h)
            out.copy_(self._pool(h, s.n, s.k))
            if kept is not None:
                kept.append(h)
        return self._summarise(src, segments, hop, widen)

    def aggregate_rows(self, src, segments, final=None, src_persistent=False):
        if not self._fused_ok(src, segments):
            # materialised form (fp32 / tf32 arithmetic, fanout > 128, wide inputs, sharded tables)
            return self._finish(self._pooled_parts(src, segments), self._combine())
        # K4: every launch of this branch is one of the library's kernels (no torch copy / convert kernels in the step)
        table = self._bf16_table(src, src_persistent)
        rows = max(s.out_row0 + s.n for s in segments)
        hmax = torch.empty((rows, self.hidden_dim), dtype=torch.float32, device=src.device)
        for s in segments:
            self._fused_hop(table, s, hmax[s.out_row0:s.out_row0 + s.n])
        s0 = segments[0]
        if len(segments) == 1 and s0.self_ids is None and s0.out_row0 == 0 and src.dtype == torch.float32:
            xs = src[s0.self_row0:s0.self_row0 + s0.n]             # the self rows are already a dense fp32 row range
        else:
            F_in = src.shape[1]
            xs = torch.empty((rows, ops.pad_cols(F_in)), dtype=torch.float32, device=src.device)[:, :F_in]
            for s in segments:
                _rows(src, s.self_ids, s.self_row0, s.n, True, out=xs[s.out_row0:s.out_row0 + s.n])
        return self._finish([(xs, self.input_dim, self.vars["self_weights"]),
                             (hmax, self.hidden_dim, self.vars["neigh_weights"])], self._combine())


class MeanPoolingAggregator(MaxPoolingAggregator):
    """act(concat_or_add(self @ Ws, mean_k(relu(neigh @ Wm + bm)) @ Wn)) - reference graphsage/aggregators.py:197-273.
    Same kernels as the max-pool aggregator with the pooling operator swapped (SURVEY section 8f row 4)."""
    pool = "mean"


class TwoMaxLayerPoolingAggregator(MaxPoolingAggregator):
    """act(concat_or_add(self @ Ws, max_k(relu(relu(neigh @ W1 + b1) @ W2 + b2)) @ Wn)) - aggregators.py:276-361: two
    Dense layers (hidden 512 / 256 "small", 1024 / 512 "big") before the max.  With bf16 math the neighbour branch is K5
    (ops.maxpool2_mlp_fused), else the materialised chain of the max-pool aggregator."""

    def __init__(self, input_dim, output_dim, model_size="small", neigh_input_dim=None, dropout=0., bias=False,
                 act=relu, name=None, concat=False, device="cuda", **kwargs):
        _SageAggregator.__init__(self, **kwargs)
        self.dropout = dropout
        self.bias = bias
        self.act = act
        self.concat = concat
        if neigh_input_dim is None:
            neigh_input_dim = input_dim
        if model_size == "small":
            self.hidden_dim_1, self.hidden_dim_2 = 512, 256
        elif model_size == "big":
            self.hidden_dim_1, self.hidden_dim_2 = 1024, 512
        else:
            raise ValueError("model_size must be 'small' or 'big'")
        self.hidden_dim = self.hidden_dim_2          # the pooled width (_summarise, the full-neighbourhood layer)
        self.math = _DEFAULT_MATH[0]
        self.mlp_layers = [Dense(input_dim=d_in, output_dim=d_out, act=relu, dropout=dropout, sparse_inputs=False,
                                 logging=self.logging, device=device, math=self.math)
                           for d_in, d_out in ((neigh_input_dim, self.hidden_dim_1),
                                               (self.hidden_dim_1, self.hidden_dim_2))]
        self.vars["neigh_weights"] = glorot([self.hidden_dim_2, output_dim], name="neigh_weights", device=device)
        self.vars["self_weights"] = glorot([input_dim, output_dim], name="self_weights", device=device)
        if self.bias:   # aggregators.py:325 reads self.output_dim before it is set; fixed as in MeanAggregator
            self.vars["bias"] = zeros([output_dim * (2 if concat else 1)], name="bias", device=device)
        self.input_dim = input_dim
        self.output_dim = output_dim
        self.neigh_input_dim = neigh_input_dim

    def _fused_ok(self, src, segments):
        return (self.math == ops.MATH_BF16 and torch.is_tensor(src) and not self.dropout and len(self.mlp_layers) == 2
                and all(fused_pool2_fits(s.k, self.neigh_input_dim, self.hidden_dim_1, self.hidden_dim_2)
                        for s in segments)
                and all(l.act is relu and "bias" in l.vars for l in self.mlp_layers))

    def _fused_hop(self, table, s, out):
        """K5 for one hop: gather -> Dense -> Dense -> max over the fanout in one wgmma kernel (bf16 operands)."""
        if getattr(self, "_packed_mlp", None) is None:
            self._packed_mlp = (ops.PackedMlpWeights(), ops.PackedMlpWeights())
        l1, l2 = (l.vars for l in self.mlp_layers)
        ops.maxpool2_mlp_fused(table, s.n, s.k, l1["weights"], l1["bias"], self._packed_mlp[0], l2["weights"], l2["bias"],
                               self._packed_mlp[1], row_ids=s.neigh_ids, row0=s.neigh_row0, K=self.neigh_input_dim,
                               out=out)


def refuse_seq_table(features):
    """The seq aggregator reads a dense fp32 table (the projection GEMM and the length rule take fp32 rows)."""
    if hasattr(features, "c_table"):
        raise NotImplementedError("the seq aggregator with a node-partitioned (ShardedFeatures) table is not implemented")
    if features is not None and features.dtype != torch.float32:
        raise NotImplementedError("the seq aggregator with a %s feature table is not implemented (float32 only)"
                                  % features.dtype)


class LSTMCell(object):
    """tf.contrib.rnn.BasicLSTMCell(H) of TF 1.8 (the reference's SeqAggregator.cell): `kernel` [K + H, 4H] - rows for the
    input first, then for h; glorot uniform, the tf.get_variable default - and `bias` [4H], zeros.  Gate columns i, j, f, o;
    the forget bias 1.0 is added at run time, not stored."""

    def __init__(self, input_dim, hidden_dim, device="cuda"):
        self.input_dim, self.hidden_dim = input_dim, hidden_dim
        self.vars = {"kernel": glorot([input_dim + hidden_dim, 4 * hidden_dim], name="kernel", device=device),
                     "bias": zeros([4 * hidden_dim], name="bias", device=device)}

    @property
    def W_x(self):
        return self.vars["kernel"][:self.input_dim]

    @property
    def W_h(self):
        return self.vars["kernel"][self.input_dim:]


class SeqAggregator(_SageAggregator):
    """act(concat_or_add(self @ Ws, h_len @ Wn)) - aggregators.py:363-449: an LSTM (`self.cell`, hidden 128 for "small",
    256 for "big") runs over the first len_i neighbours of each node, len_i = max(1, number of neighbour rows that are not
    all zero), and h after len_i steps is the neighbour summary.  The input projection X W_x + b is the library GEMM
    (self.math), the recurrence the fp32 kernels gs_lstm_forward / gs_seq_lengths.  `dropout` is kept but never applied:
    the reference's SeqAggregator._call draws no mask."""

    def __init__(self, input_dim, output_dim, model_size="small", neigh_input_dim=None, dropout=0., bias=False, act=relu,
                 name=None, concat=False, device="cuda", **kwargs):
        super(SeqAggregator, self).__init__(**kwargs)
        self.dropout = dropout
        self.bias = bias
        self.act = act
        self.concat = concat
        if neigh_input_dim is None:
            neigh_input_dim = input_dim
        if model_size == "small":
            hidden_dim = self.hidden_dim = 128
        elif model_size == "big":
            hidden_dim = self.hidden_dim = 256
        else:
            raise ValueError("model_size must be 'small' or 'big'")
        self.vars["neigh_weights"] = glorot([hidden_dim, output_dim], name="neigh_weights", device=device)
        self.vars["self_weights"] = glorot([input_dim, output_dim], name="self_weights", device=device)
        if self.bias:   # aggregators.py:395 reads self.output_dim before it is set; fixed as in MeanAggregator
            self.vars["bias"] = zeros([output_dim * (2 if concat else 1)], name="bias", device=device)
        self.input_dim = input_dim
        self.output_dim = output_dim
        self.neigh_input_dim = neigh_input_dim
        self.math = _DEFAULT_MATH[0]
        self.cell = LSTMCell(neigh_input_dim, hidden_dim, device=device)

    def _neigh_hidden(self, X, n, k, out=None, kept=None):
        """h after len_i steps over the n sequences of k rows of X [n*k, neigh_input_dim]; `kept` (training) receives X,
        the lengths, the gates, c and h_{t-1}."""
        lengths = ops.seq_lengths(X, n, k)
        if getattr(self.cell, "_packed", None) is None:
            self.cell._packed = ops.PackedWeights()
        P = ops.sage_gemm([(X, self.neigh_input_dim, self.cell.W_x)], bias=self.cell.vars["bias"], math=self.math,
                          packed=self.cell._packed)
        if kept is None:
            return ops.lstm_forward(P, self.cell.W_h, lengths, n, k, out=out)
        h, gates, c, h_prev = ops.lstm_forward(P, self.cell.W_h, lengths, n, k, out=out, train=True)
        kept += [X, lengths, gates, c, h_prev]
        return h

    def _call(self, inputs):
        self_vecs, neigh_vecs = inputs
        n, k, d = neigh_vecs.shape
        h = self._neigh_hidden(neigh_vecs.reshape(n * k, d), n, k)
        return self._finish([(self_vecs, self.input_dim, self.vars["self_weights"]),
                             (h, self.hidden_dim, self.vars["neigh_weights"])], self._combine())

    def _seq_parts(self, src, segments, kept=None):
        refuse_seq_table(src)
        return self._summarise(src, segments, lambda i, s, out: self._neigh_hidden(
            _rows(src, s.neigh_ids, s.neigh_row0, s.n * s.k), s.n, s.k, out=out, kept=kept))

    def aggregate_rows(self, src, segments, final=None, src_persistent=False):
        return self._finish(self._seq_parts(src, segments), self._combine())
