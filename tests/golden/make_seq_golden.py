"""Generate tests/golden/seq.npz - the LSTM sequence aggregator - by executing the reference's own SeqAggregator
(graphsage/aggregators.py:363-449) and SampleAndAggregate.aggregate (graphsage/models.py:278-330) under the numpy TF
shim.  Same rules as make_golden.py (whose shim set-up, reference imports and helpers it reuses): run where the reference
lies; nothing from it is copied.

The shim gains here the few TF 1.8 symbols SeqAggregator._call touches: tf.contrib.rnn.BasicLSTMCell and tf.nn.dynamic_rnn,
restated from TF 1.8's documented semantics (gate columns i, j, f, o of [x, h] @ kernel + bias, forget bias 1.0 added at
run time; with sequence_length the state is frozen and the outputs are zero past the length), and sign, abs, maximum,
range, gather, and get_shape() on the RNN outputs.  The cell's internals are thus pinned by the TF formula, not by running
TF; the aggregator's own lines (length rule, output gather, combination) are the reference's.

    python tests/golden/make_seq_golden.py
"""
import types

import numpy as np

import make_golden as mg            # installs the shim and imports the reference's modules
from make_golden import SAGEInfo, SampleAndAggregate, UniformNeighborSampler, _Stub, save, tf, tf_shim


class _Shaped(np.ndarray):
    """An ndarray that answers t.get_shape()[i] like a TF tensor (aggregators.py:430)."""

    def get_shape(self):
        return list(self.shape)


def _sigmoid(x):
    return 1.0 / (1.0 + np.exp(-x))


KERNEL_SEED = [1000]


class BasicLSTMCell(object):
    """TF 1.8 tf.contrib.rnn.BasicLSTMCell(num_units, forget_bias=1.0): variables made on the first call - kernel
    [input + num_units, 4 num_units] by get_variable's default (glorot uniform), bias [4 num_units] zeros - and reused.
    The kernel is drawn by oracle.seq.cell_kernel from the next seed of KERNEL_SEED, so the fixture stores the seed (a
    few bytes) instead of the incompressible [K + H, 4H] values."""

    def __init__(self, num_units, forget_bias=1.0, **k):
        self.num_units, self.forget_bias = num_units, forget_bias
        self.kernel = self.bias = self.kernel_seed = None

    def zero_state(self, batch_size, dtype):
        z = np.zeros((batch_size, self.num_units), dtype)
        return (z, z.copy())

    def __call__(self, x, state):
        H = self.num_units
        if self.kernel is None:
            from oracle.seq import cell_kernel
            self.kernel_seed = KERNEL_SEED[0]
            KERNEL_SEED[0] += 1
            self.kernel = cell_kernel(self.kernel_seed, (x.shape[1] + H, 4 * H))
            self.bias = np.zeros(4 * H, np.float32)
        c, h = state
        z = np.concatenate([x, h], axis=1) @ self.kernel + self.bias
        i, j, f, o = z[:, :H], z[:, H:2 * H], z[:, 2 * H:3 * H], z[:, 3 * H:]
        c = c * _sigmoid(f + self.forget_bias) + _sigmoid(i) * np.tanh(j)
        h = np.tanh(c) * _sigmoid(o)
        return h, (c, h)


def dynamic_rnn(cell, inputs, sequence_length=None, initial_state=None, dtype=None, time_major=False, **k):
    """TF 1.8 tf.nn.dynamic_rnn (batch major): past sequence_length[b] the state of b is copied through and its output
    is zero."""
    x = np.asarray(inputs, np.float32)
    n, steps, _ = x.shape
    state = initial_state if initial_state is not None else cell.zero_state(n, np.float32)
    lengths = np.full(n, steps) if sequence_length is None else np.asarray(sequence_length)
    outs = np.zeros((n, steps, cell.num_units), np.float32)
    for t in range(steps):
        out, new = cell(x[:, t], state)
        on = (t < lengths)[:, None]
        outs[:, t] = np.where(on, out, 0)
        state = tuple(np.where(on, a, b) for a, b in zip(new, state))
    return outs.view(_Shaped), state


DROPOUT_CALLS = [0]


def _install_rnn():
    tf.contrib.rnn = types.SimpleNamespace(BasicLSTMCell=BasicLSTMCell)
    tf.nn.dynamic_rnn = dynamic_rnn
    dropout = tf.nn.dropout

    def counting_dropout(x, keep_prob, **k):
        DROPOUT_CALLS[0] += 1
        return dropout(x, keep_prob, **k)

    tf.nn.dropout = counting_dropout
    tf.sign = lambda x: np.sign(np.asarray(x))
    tf.abs = lambda x: np.abs(np.asarray(x))
    tf.maximum = lambda a, b: np.maximum(np.asarray(a), np.asarray(b))
    tf.range = lambda start, limit=None, delta=1, **k: np.arange(start, limit, delta, dtype=np.int32)
    tf.gather = lambda params, indices, **k: np.asarray(params)[np.asarray(indices).astype(np.int64)]


def _seq_class(output_dim):
    """The reference's SeqAggregator with output_dim set before __init__ runs: its bias=True branch reads
    self.output_dim before assigning it (aggregators.py:394-395)."""
    from graphsage.aggregators import SeqAggregator
    return type("SeqAggregator", (SeqAggregator,), {"output_dim": output_dim})


def golden_seq():
    _install_rnn()
    r = np.random.RandomState(11)
    n, k, din, dout = 9, 5, 12, 6
    selfv = r.randn(n, din).astype(np.float32)
    neigh = r.randn(n, k, din).astype(np.float32)
    neigh[1, 1] = 0.0                       # an interspersed zero row: len 4, position 4 is never read
    neigh[2] = 0.0                          # an all-zero sequence: len clamps to 1
    neigh[3, 3:] = 0.0                      # trailing zero rows (the dummy row's padding): len 3
    neigh[4, 0] = -0.0                      # a row of negative zeros counts as zero
    neigh[5, :, 1:] = 0.0                   # rows with a single non-zero element count
    out = {"self": selfv, "neigh": neigh}
    for tag, concat, bias, size in (("c0", False, False, "small"), ("c1", True, False, "small"),
                                    ("bias", False, True, "small"), ("big", True, False, "big")):
        DROPOUT_CALLS[0] = 0
        agg = _seq_class(dout)(din, dout, model_size=size, bias=bias, concat=concat, dropout=0.5)
        out[tag + "_out"] = np.asarray(agg((selfv, neigh)))
        out[tag + "_nw"], out[tag + "_sw"] = agg.vars["neigh_weights"], agg.vars["self_weights"]
        out[tag + "_kernel_seed"], out[tag + "_kernel_shape"] = np.int64(agg.cell.kernel_seed), np.array(agg.cell.kernel.shape)
        out[tag + "_cell_bias"] = agg.cell.bias
        if bias:
            out[tag + "_bias"] = agg.vars["bias"]
        out[tag + "_dropout_calls"] = np.int32(DROPOUT_CALLS[0])
    # 2-layer K-hop: the reference's aggregate() with SeqAggregator; node 3's neighbours are all the dummy id
    nn, md, f, B = 60, 8, 10, 6
    adj = r.randint(0, nn, size=(nn + 1, md)).astype(np.int32)
    adj[nn, :] = nn
    adj[3, :] = nn
    feats = np.vstack([r.randn(nn, f).astype(np.float32), np.zeros((1, f), np.float32)])
    seeds = r.randint(0, nn, size=B).astype(np.int32)
    seeds[0] = 3
    dims, fan = [f, 8, 5], [4, 3]
    from graphsage.aggregators import SeqAggregator
    tf_shim.SHUFFLE_SEED, tf_shim.SHUFFLE_COUNTER = 123, 40
    sampler = UniformNeighborSampler(adj)
    infos = [SAGEInfo("node", sampler, fan[i], dims[i + 1]) for i in range(len(fan))]
    stub = _Stub()
    stub.batch_size = B
    stub.aggregator_cls = SeqAggregator
    stub.placeholders = {"dropout": 0.0}
    samples, support = SampleAndAggregate.sample(stub, seeds, infos)
    hidden, aggs = SampleAndAggregate.aggregate(stub, samples, feats, dims, fan, support, concat=True)
    out.update(khop_adj=adj, khop_feats=feats, khop_seeds=seeds, khop_dims=np.array(dims), khop_fanout=np.array(fan),
               khop_support=np.array(support), khop_out=np.asarray(hidden))
    for h, s in enumerate(samples):
        out["khop_samples%d" % h] = np.asarray(s).astype(np.int32)
    for li, a in enumerate(aggs):
        out["khop_L%d_nw" % li], out["khop_L%d_sw" % li] = a.vars["neigh_weights"], a.vars["self_weights"]
        out["khop_L%d_kernel_seed" % li] = np.int64(a.cell.kernel_seed)
        out["khop_L%d_kernel_shape" % li] = np.array(a.cell.kernel.shape)
        out["khop_L%d_cell_bias" % li] = a.cell.bias
    save("seq", **out)


if __name__ == "__main__":
    mg._standalone(golden_seq)
