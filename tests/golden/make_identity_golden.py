"""Generate tests/golden/identity.npz - trainable node embeddings (identity_dim > 0) - by executing the reference's own
constructor lines (graphsage/supervised_models.py:51-67, graphsage/models.py:229-245) with build() stubbed out, then its
aggregate(), under the numpy TF shim, with features and without (features=None).  Same rules as make_golden.py (whose
shim set-up, reference imports and helpers it reuses): run where the reference lies; nothing from it is copied.

    python tests/golden/make_identity_golden.py
"""
import types

import numpy as np

import make_golden as mg            # installs the shim and imports the reference's modules
from make_golden import SAGEInfo, SampleAndAggregate, UniformNeighborSampler, save, tf_shim


class _Tensor(np.ndarray):
    """An ndarray that also answers t.get_shape().as_list(): the reference sizes node_embeddings from the adjacency
    tensor that way (models.py:230, supervised_models.py:52)."""

    def get_shape(self):
        return types.SimpleNamespace(as_list=lambda: list(self.shape))


def golden_identity():
    from graphsage.supervised_models import SupervisedGraphsage as RefSupervised

    class SupervisedNoBuild(RefSupervised):
        def build(self):
            pass

    class UnsupervisedNoBuild(SampleAndAggregate):
        def build(self):
            pass

    r = np.random.RandomState(43)
    n, md, f, d, B = 120, 16, 10, 6, 7
    adj = r.randint(0, n, size=(n + 1, md)).astype(np.int32)
    adj[n, :] = n
    adj[5, :] = n                                       # a node whose samples are all the padding id
    feats = np.vstack([r.randn(n, f).astype(np.float32), np.zeros((1, f), np.float32)])   # supervised_train.py:133-135
    seeds = r.randint(0, n, size=B).astype(np.int32)
    seeds[0] = 5
    fan, dims_out = [4, 3], [8, 5]
    out = dict(adj=adj, feats=feats, seeds=seeds, fanout=np.array(fan), identity_dim=np.int32(d))
    for model, cls in (("sup", SupervisedNoBuild), ("unsup", UnsupervisedNoBuild)):
        for tag, features in (("feat", feats), ("nofeat", None)):
            key = "%s_%s_" % (model, tag)
            tf_shim.SHUFFLE_SEED, tf_shim.SHUFFLE_COUNTER = 123, 40
            sampler = UniformNeighborSampler(adj)
            infos = [SAGEInfo("node", sampler, fan[i], dims_out[i]) for i in range(len(fan))]
            ph = {"batch": seeds, "batch1": seeds, "batch2": seeds, "batch_size": B, "dropout": 0.0}
            args = (ph, features, adj.view(_Tensor), None, infos)
            m = cls(3, *args, identity_dim=d) if model == "sup" else cls(*args, identity_dim=d)
            samples, support = m.sample(seeds, infos)
            # a one-element params list of tf.nn.embedding_lookup is the table itself (as in make_golden.golden_khop)
            hidden, aggs = m.aggregate(samples, m.features, m.dims, fan, support, concat=m.concat)
            out[key + "embeds"] = np.asarray(m.embeds)
            out[key + "features"] = np.asarray(m.features)
            out[key + "dims"] = np.array(m.dims)
            out[key + "out"] = np.asarray(hidden)
            for li, a in enumerate(aggs):
                for name, v in a.vars.items():
                    out["%sL%d_%s" % (key, li, name)] = v
    save("identity", **out)


if __name__ == "__main__":
    mg._standalone(golden_identity)
