"""Generate tests/golden/twomax.npz - the two-layer max-pool aggregator - by executing the reference's own
TwoMaxLayerPoolingAggregator (graphsage/aggregators.py:276-361), layers.Dense and SampleAndAggregate.sample / .aggregate
(graphsage/models.py:254-330) under the numpy TF shim.  Same rules as make_golden.py (whose shim set-up, reference
imports and helpers it reuses): run where the reference lies; nothing from it is copied.

Here (tf_shim.py itself is unchanged) every variable the reference draws - glorot (inits.py:15-19) and Dense's
xavier get_variable (layers.py:96-99), both U(-r, r) with r = sqrt(6 / (fan_in + fan_out)) - comes from the next seed of
WEIGHT_SEED through oracle.seq.cell_kernel, so the fixture stores seeds and shapes, not the megabytes of a "big" W1.
The Dense biases are made non-zero after construction (stored: they are small).  The reference's bias=True branch reads
self.output_dim before assigning it (aggregators.py:325-326), so the class is given output_dim before __init__ runs;
its bias has width output_dim whatever concat is, so bias=True is recorded without concat (with concat it cannot run).
One dropout pass replaces tf.nn.dropout by a stand-in that draws each call's mask from oracle/dropout.py with the next
call number and records the shape of every dropped tensor (as make_dropout_golden.py does): it pins the mlp -> mlp2 call
order and the [n*k, .] element layout of both sites.

    python tests/golden/make_twomax_golden.py
"""
import numpy as np

import make_golden as mg            # installs the shim and imports the reference's modules
from make_golden import SAGEInfo, SampleAndAggregate, UniformNeighborSampler, save, tf, tf_shim
from oracle import dropout as odrop
from oracle.seq import cell_kernel

WEIGHT_SEED = [5000]
DRAWS = []                           # (seed, rows, cols) of every variable drawn, in order
BIAS_RNG = np.random.RandomState(77)
RATE, DROP_SEED = 0.5, 20261017
_CALLS = []


def _draw(shape):
    seed = WEIGHT_SEED[0]
    WEIGHT_SEED[0] += 1
    DRAWS.append((seed,) + tuple(int(s) for s in shape))
    return cell_kernel(seed, shape)


def _random_uniform(shape, minval=0.0, maxval=1.0, dtype=np.float32, **k):
    r = np.sqrt(6.0 / (shape[0] + shape[1]))
    assert np.isclose(maxval, r) and np.isclose(minval, -r), "only glorot draws are expected"
    return _draw(shape)


def _get_variable(name, shape=None, dtype=np.float32, initializer=None, regularizer=None, **k):
    return _draw(tuple(shape))


def _dropout(x, keep_prob, **k):
    x = np.asarray(x, dtype=np.float32)
    if float(keep_prob) == 1.0:
        return x
    assert np.float32(1.0 - keep_prob) == np.float32(RATE)
    y = odrop.apply_nd(x, DROP_SEED, len(_CALLS), RATE)
    _CALLS.append(x.shape)
    return y


def _cls(output_dim):
    """The reference's class with output_dim preset, and non-zero Dense biases drawn right after construction."""
    from graphsage.aggregators import TwoMaxLayerPoolingAggregator

    def __init__(self, *a, **k):
        TwoMaxLayerPoolingAggregator.__init__(self, *a, **k)
        for layer in self.mlp_layers:
            layer.vars["bias"] = (BIAS_RNG.randn(*layer.vars["bias"].shape) * 0.1).astype(np.float32)

    return type("TwoMaxLayerPoolingAggregator", (TwoMaxLayerPoolingAggregator,), {"output_dim": output_dim,
                                                                                  "__init__": __init__})


def _record(out, key, agg, first_draw):
    out[key + "draws"] = np.array(DRAWS[first_draw:], np.int64)      # W1, W2, neigh_weights, self_weights in order
    out[key + "b1"], out[key + "b2"] = agg.mlp_layers[0].vars["bias"], agg.mlp_layers[1].vars["bias"]
    if "bias" in agg.vars:
        out[key + "bias"] = agg.vars["bias"]


def golden_twomax():
    tf.random_uniform = _random_uniform
    tf.get_variable = _get_variable
    tf.nn.dropout = _dropout
    r = np.random.RandomState(12)
    n, k, din, dout = 7, 4, 10, 6
    selfv = r.randn(n, din).astype(np.float32)
    neigh = r.randn(n, k, din).astype(np.float32)
    neigh[2] = 0.0                          # every neighbour is the dummy row (zero features)
    out = {"self": selfv, "neigh": neigh}
    for tag, concat, bias, size in (("c0", False, False, "small"), ("c1", True, False, "small"),
                                    ("bias", False, True, "small"), ("big", True, False, "big")):
        first = len(DRAWS)
        agg = _cls(dout)(din, dout, model_size=size, bias=bias, concat=concat)
        out[tag + "_out"] = np.asarray(agg((selfv, neigh)))
        _record(out, tag + "_", agg, first)
    # two layers, concat: sample / aggregate with the class; node 3's neighbours are all the dummy id
    nn, md, f, B = 60, 8, 10, 6
    adj = r.randint(0, nn, size=(nn + 1, md)).astype(np.int32)
    adj[nn, :] = nn
    adj[3, :] = nn
    feats = np.vstack([r.randn(nn, f).astype(np.float32), np.zeros((1, f), np.float32)])
    seeds = r.randint(0, nn, size=B).astype(np.int32)
    seeds[0] = 3
    dims, fan = [f, 8, 5], [4, 3]
    out.update(khop_adj=adj, khop_feats=feats, khop_seeds=seeds, khop_dims=np.array(dims), khop_fanout=np.array(fan))
    for tag, rate in (("khop", 0.0), ("drop", RATE)):
        tf_shim.SHUFFLE_SEED, tf_shim.SHUFFLE_COUNTER = 123, 40
        sampler = UniformNeighborSampler(adj)
        infos = [SAGEInfo("node", sampler, fan[i], dims[i + 1]) for i in range(len(fan))]
        stub = mg._Stub()
        stub.batch_size, stub.aggregator_cls, stub.placeholders = B, _cls(None), {"dropout": rate}
        samples, support = SampleAndAggregate.sample(stub, seeds, infos)
        del _CALLS[:]
        first = len(DRAWS)
        hidden, aggs = SampleAndAggregate.aggregate(stub, samples, feats, dims, fan, support, concat=True,
                                                    model_size="small")
        out[tag + "_out"], out[tag + "_support"] = np.asarray(hidden), np.array(support)
        for h, s in enumerate(samples):
            out["%s_samples%d" % (tag, h)] = np.asarray(s).astype(np.int32)
        per = len(DRAWS[first:]) // len(aggs)
        for li, a in enumerate(aggs):
            _record(out, "%s_L%d_" % (tag, li), a, first + li * per)
            out["%s_L%d_draws" % (tag, li)] = out["%s_L%d_draws" % (tag, li)][:per]
        if rate:
            calls = -np.ones((len(_CALLS), 3), np.int64)
            for i, s in enumerate(_CALLS):
                calls[i, :len(s)] = s
            out[tag + "_calls"], out[tag + "_rate"], out[tag + "_seed"] = calls, np.float32(RATE), np.uint64(DROP_SEED)
    save("twomax", **out)


if __name__ == "__main__":
    mg._standalone(golden_twomax)
