"""Generate tests/golden/full_neighbor.npz - full-neighbourhood embeddings written by the reference's own sampled path.
Executes the reference's SampleAndAggregate.sample / .aggregate and aggregators (graphsage/models.py:254-330,
aggregators.py) under the numpy TF shim (tf_shim.py) on a d-regular graph with max_degree = d and every layer's
num_samples = d.  Every padded row is then a permutation of the node's neighbours and the sampler draws all of them, so
the reference's sampled result is the full-neighbourhood result up to summation order.  Run where the reference lies;
nothing from it is copied.

    python tests/golden/make_full_neighbor_golden.py

Cases (two layers each): mean, gcn, maxpool, meanpool; concat off and on (gcn: off - its single weight ignores concat).
Keys per case <c>: <c>_dims, <c>_concat, <c>_L<l>_<var> (weights as the oracle's dicts name them), <c>_out (the
l2-normalised embeddings of nodes 0 .. N-1).  Shared: feats [N+1, F] (row N zero), indptr, indices.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
sys.path.insert(0, "/root/reference")

import tf_shim  # noqa: E402

tf = tf_shim.install()

from graphsage.aggregators import GCNAggregator, MaxPoolingAggregator, MeanAggregator, MeanPoolingAggregator  # noqa: E402
from graphsage.models import SAGEInfo, SampleAndAggregate  # noqa: E402
from graphsage.neigh_samplers import UniformNeighborSampler  # noqa: E402

N, D, F = 48, 4, 12
OFFSETS = (1, 2, 5)          # node v's neighbours: v +- 1, v + 2, v - 5 (mod N) -> 4-regular, duplicate-free


def regular_csr(rs):
    """CSR of a d-regular graph; each row's order is shuffled so CSR order differs from any padded order."""
    rows = []
    for v in range(N):
        nb = np.array([(v + 1) % N, (v - 1) % N, (v + 2) % N, (v - 5) % N])
        rows.append(nb[rs.permutation(D)])
    indptr = np.arange(N + 1, dtype=np.int64) * D
    return indptr, np.concatenate(rows).astype(np.int32)


class _Stub(object):
    """Just the attributes SampleAndAggregate.sample/.aggregate read (models.py:254-330)."""


def agg_vars(a, kind):
    out = dict(a.vars)
    if kind == "gcn":
        out = {"weights": a.vars["weights"]}
    if hasattr(a, "mlp_layers"):
        out["mlp_weights"] = a.mlp_layers[0].vars["weights"]
        out["mlp_bias"] = a.mlp_layers[0].vars["bias"]
    return out


def main():
    rs = np.random.RandomState(11)
    indptr, indices = regular_csr(rs)
    adj = np.full((N + 1, D), N, dtype=np.int32)
    for v in range(N):
        adj[v] = rs.permutation(indices[indptr[v]:indptr[v + 1]])      # a padded row: another order of the same row
    feats = np.vstack([rs.randn(N, F).astype(np.float32), np.zeros((1, F), np.float32)])
    out = {"feats": feats, "indptr": indptr, "indices": indices}
    seeds = np.arange(N, dtype=np.int32)
    cases = []
    for kind, cls in (("mean", MeanAggregator), ("gcn", GCNAggregator), ("maxpool", MaxPoolingAggregator),
                      ("meanpool", MeanPoolingAggregator)):
        for concat in ((False,) if kind == "gcn" else (False, True)):
            name = "%s_c%d" % (kind, concat)
            dims = [F, 10, 6]
            tf_shim.SHUFFLE_SEED, tf_shim.SHUFFLE_COUNTER = 5, 0
            sampler = UniformNeighborSampler(adj)
            infos = [SAGEInfo("node", sampler, D, dims[i + 1]) for i in range(2)]
            stub = _Stub()
            stub.batch_size = N
            stub.aggregator_cls = cls
            stub.placeholders = {"dropout": 0.0}
            samples, support = SampleAndAggregate.sample(stub, seeds, infos)
            for h in range(1, 3):                                   # every sample is a whole row
                s = np.asarray(samples[h]).reshape(-1, D)
                parents = np.asarray(samples[h - 1]).reshape(-1)
                for p, row in zip(parents, s):
                    assert sorted(row) == sorted(indices[indptr[p]:indptr[p + 1]])
            hidden, aggs = SampleAndAggregate.aggregate(stub, samples, feats, dims, [D, D], support, concat=concat)
            out[name + "_dims"] = np.array(dims)
            out[name + "_concat"] = concat
            out[name + "_out"] = np.asarray(tf.nn.l2_normalize(hidden, 1), dtype=np.float32)     # models.py:368
            for li, a in enumerate(aggs):
                for key, v in agg_vars(a, kind).items():
                    out["%s_L%d_%s" % (name, li, key)] = np.asarray(v, dtype=np.float32)
            cases.append(name)
    out["cases"] = np.array(cases)
    path = os.path.join(HERE, "full_neighbor.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, cases)


if __name__ == "__main__":
    main()
