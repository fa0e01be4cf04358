"""Generate tests/golden/dropout.npz - training dropout - by executing the reference's own models.aggregate, aggregators,
layers.Dense (the supervised head, supervised_models.py:88-92) and the unsupervised three-pass order (models.py:347-360)
under the numpy TF shim, with tf.nn.dropout replaced here (tf_shim.py itself is unchanged) by a stand-in that draws each
call's mask from oracle/dropout.py with the next call number and records the shape of every dropped tensor.  Same rules as
make_golden.py (whose shim set-up, reference imports and helpers it reuses): run where the reference lies; nothing from it
is copied.

    python tests/golden/make_dropout_golden.py
"""
import numpy as np

import make_golden as mg            # installs the shim and imports the reference's modules
from make_golden import SAGEInfo, SampleAndAggregate, UniformNeighborSampler, save, tf, tf_shim
from oracle import dropout as odrop

RATE, SEED = 0.5, 20261015
_CALLS = []                          # shape of every dropped tensor, in call order


def _dropout(x, keep_prob, **k):
    x = np.asarray(x, dtype=np.float32)
    assert np.float32(1.0 - keep_prob) == np.float32(RATE)
    y = odrop.apply_nd(x, SEED, len(_CALLS), RATE)
    _CALLS.append(x.shape)
    return y


def _shapes(calls):
    """[n_calls, 3] int64, shapes padded with -1."""
    out = -np.ones((len(calls), 3), dtype=np.int64)
    for i, s in enumerate(calls):
        out[i, :len(s)] = s
    return out


def golden_dropout():
    from graphsage.aggregators import GCNAggregator, MaxPoolingAggregator, MeanAggregator, MeanPoolingAggregator
    from graphsage.layers import Dense
    tf.nn.dropout = _dropout
    r = np.random.RandomState(47)
    n, md, f, B, NEG, C = 60, 12, 9, 5, 4, 3
    adj = r.randint(0, n, size=(n + 1, md)).astype(np.int32)
    adj[n, :] = n
    feats = np.vstack([r.randn(n, f).astype(np.float32), np.zeros((1, f), np.float32)])
    seeds = r.randint(0, n, size=B).astype(np.int32)
    neg = r.randint(0, n, size=NEG).astype(np.int32)
    fan, dims = [3, 2], [f, 7, 4]
    out = dict(adj=adj, feats=feats, seeds=seeds, neg=neg, fanout=np.array(fan), dims=np.array(dims), rate=np.float32(RATE),
               seed=np.uint64(SEED))
    kinds = [("mean", MeanAggregator), ("gcn", GCNAggregator), ("maxpool", MaxPoolingAggregator),
             ("meanpool", MeanPoolingAggregator)]
    for kind, cls in kinds:
        for concat in ((False,) if kind == "gcn" else (False, True)):      # GCN's output is never concatenated
            key = "%s_c%d_" % (kind, int(concat))
            stub = mg._Stub()
            stub.batch_size, stub.aggregator_cls, stub.placeholders = B, cls, {"dropout": RATE}
            passes = []
            for tag, ids, bs in (("sup", seeds, B), ("u1", seeds, B), ("u2", seeds[::-1].copy(), B), ("un", neg, NEG)):
                tf_shim.SHUFFLE_SEED, tf_shim.SHUFFLE_COUNTER = 123, 40
                sampler = UniformNeighborSampler(adj)
                infos = [SAGEInfo("node", sampler, fan[i], dims[i + 1]) for i in range(len(fan))]
                samples, support = SampleAndAggregate.sample(stub, ids, infos, bs)
                passes.append((tag, samples, support, bs))
            # supervised: one aggregate pass, l2_normalize, then the head Dense with dropout (supervised_models.py:79-92)
            del _CALLS[:]
            tag, samples, support, bs = passes[0]
            hidden, aggs = SampleAndAggregate.aggregate(stub, samples, feats, dims, fan, support, batch_size=bs, concat=concat,
                                                        model_size="small")
            dim_mult = 2 if concat else 1
            head = Dense(dim_mult * dims[-1], C, dropout=RATE, act=lambda x: x)
            logits = head(tf.nn.l2_normalize(hidden, 1))
            out[key + "sup_out"], out[key + "sup_logits"] = hidden, logits
            out[key + "head_w"], out[key + "head_b"] = head.vars["weights"], head.vars["bias"]
            out[key + "sup_calls"] = _shapes(_CALLS)
            for h, s in enumerate(samples):
                out["%ssup_samples%d" % (key, h)] = np.asarray(s).astype(np.int32)
            for li, a in enumerate(aggs):
                for name, v in a.vars.items():
                    out["%sL%d_%s" % (key, li, name)] = v
                if hasattr(a, "mlp_layers"):
                    out["%sL%d_mlp_weights" % (key, li)] = a.mlp_layers[0].vars["weights"]
                    out["%sL%d_mlp_bias" % (key, li)] = a.mlp_layers[0].vars["bias"]
            # unsupervised: batch1, batch2, negatives through the same aggregators, fresh draws per pass (models.py:347-360)
            del _CALLS[:]
            for tag, samples, support, bs in passes[1:]:
                o, _ = SampleAndAggregate.aggregate(stub, samples, feats, dims, fan, support, batch_size=bs, aggregators=aggs,
                                                    concat=concat, model_size="small")
                out[key + tag + "_out"] = o
                for h, s in enumerate(samples):
                    out["%s%s_samples%d" % (key, tag, h)] = np.asarray(s).astype(np.int32)
            out[key + "unsup_calls"] = _shapes(_CALLS)
    save("dropout", **out)


if __name__ == "__main__":
    mg._standalone(golden_dropout)
