"""Generate tests/golden/n2v.npz - the Node2Vec / DeepWalk baseline - by executing the reference's own
Node2VecModel._build, _loss and _accuracy (graphsage/models.py:408-501) under the numpy TF shim, with build() /
_minimize stubbed out (no optimizer runs under the shim) and the tables replaced by seeded RandomState values.
tf.nn.fixed_unigram_candidate_sampler draws from oracle/node2vec.py (TF's stream is unobtainable); it and the few other
symbols the shim lacks are patched in here, so tf_shim.py and the other fixtures are untouched.  Same rules as
make_golden.py (whose shim set-up and helpers it reuses): run where the reference lies; nothing from it is copied.

    python tests/golden/make_n2v_golden.py
"""
import numpy as np

import make_golden as mg            # installs the shim and imports the reference's modules
from make_golden import save, tf, tf_shim
from oracle import node2vec as on2v

_SAMPLER = {}                        # (seed, counter) of the next sampler call, and the arguments it was called with


def _fixed_unigram_candidate_sampler(true_classes, num_true, num_sampled, unique, range_max, distortion, unigrams, **k):
    _SAMPLER["args"] = dict(num_true=num_true, unique=unique, range_max=range_max, distortion=distortion)
    assert len(unigrams) == range_max
    ids = on2v.sample_unigram_unique(np.asarray(unigrams), num_sampled, _SAMPLER["seed"], _SAMPLER["counter"],
                                     distortion=distortion)
    return ids.astype(np.int64), None, None


def _install():
    tf.nn.fixed_unigram_candidate_sampler = _fixed_unigram_candidate_sampler
    tf.truncated_normal = lambda shape, stddev=1.0, **k: np.clip(
        tf_shim.INIT_RNG.normal(0.0, stddev, size=shape), -2 * stddev, 2 * stddev).astype(np.float32)
    tf.multiply = lambda a, b: np.asarray(a) * np.asarray(b)
    tf.train.GradientDescentOptimizer = lambda learning_rate=None, **k: None


def golden_n2v():
    from graphsage.models import Node2VecModel as RefNode2Vec

    class Node2VecNoBuild(RefNode2Vec):
        def build(self):
            pass

    _install()
    r = np.random.RandomState(53)
    out = {}
    # case 0: a short batch (B = 13) with duplicates in batch1, batch2 and across batch2 and the negatives;
    # case 1: a wider table, B = 37, d = 50 (the reference's default nodevec_dim)
    for ci, (V, d, S, B, seed, counter) in enumerate([(40, 8, 6, 13, 7, 3), (300, 50, 20, 37, 11, 1 << 33)]):
        deg = r.randint(0, 12, size=V).astype(np.float64)
        deg[0] = 0.0                                            # an id that can never be a negative
        deg[1] = 40.0                                           # a hub: many rejections
        T = r.uniform(-1, 1, size=(V, d)).astype(np.float32)
        C = (r.randn(V, d) / np.sqrt(d)).astype(np.float32)
        b = (r.randn(V) * 0.3).astype(np.float32)
        neg = on2v.sample_unigram_unique(deg, S, seed, counter)
        batch1 = r.randint(0, V, size=B).astype(np.int32)
        batch2 = r.randint(0, V, size=B).astype(np.int32)
        batch1[1] = batch1[0]                                   # duplicates in batch1
        batch2[2] = batch2[3] = batch2[4]                       # ... in batch2
        batch2[5], batch2[6] = neg[0], neg[S - 1]               # ... across batch2 and the negatives
        ph = {"batch1": batch1, "batch2": batch2, "batch_size": B, "dropout": 0.0}
        tf.app.flags.FLAGS.neg_sample_size = S
        m = Node2VecNoBuild(ph, V, deg, nodevec_dim=d, lr=0.01)
        m.target_embeds, m.context_embeds, m.context_bias = T, C, b
        _SAMPLER.update(seed=seed, counter=counter)
        m._build()
        m._loss()
        m._accuracy()
        assert _SAMPLER["args"] == dict(num_true=1, unique=True, range_max=V, distortion=0.75), _SAMPLER["args"]
        assert np.array_equal(np.asarray(m.neg_samples), neg)
        key = "c%d_" % ci
        out.update({key + "deg": deg, key + "T": T, key + "C": C, key + "b": b, key + "batch1": batch1,
                    key + "batch2": batch2, key + "neg": neg, key + "seed": np.uint64(seed), key + "counter": np.uint64(counter),
                    key + "loss": np.float64(m.loss), key + "aff_all": np.asarray(m.aff_all),
                    key + "ranks": np.asarray(m.ranks), key + "mrr": np.float64(m.mrr),
                    key + "outputs1": np.asarray(m.outputs1)})
    out["n_cases"] = np.int32(2)
    save("n2v", **out)


if __name__ == "__main__":
    mg._standalone(golden_n2v)
