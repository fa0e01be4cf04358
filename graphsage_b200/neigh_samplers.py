"""UniformNeighborSampler - the surface of reference graphsage/neigh_samplers.py:15-29 over the
K1 sampler kernels."""
import torch

from . import ops
from .layers import Layer


class UniformNeighborSampler(Layer):
    """Uniformly samples neighbours.  Assumes adj lists are padded with random re-sampling
    (reference graphsage/minibatch.py:227-245).

    sampler((ids, num_samples)) -> int32 [n, num_samples] with out[i, j] = adj_info[ids[i], pi[j]] for ONE
    column permutation pi per call (neigh_samplers.py:26-28).  pi comes from Philox4x32-10 keyed by
    `seed`, counter = number of calls so far (oracle/sampler.py documents the contract).
    """

    def __init__(self, adj_info, seed=123, **kwargs):
        super(UniformNeighborSampler, self).__init__(**kwargs)
        self.set_adj(adj_info)
        self.seed = int(seed)
        self.counter = 0          # one fresh permutation per call, like a new random_shuffle op execution
        self.counter_dev = None   # optional device uint64 added to `counter` (CUDA-graph replay)

    def set_adj(self, adj_info):
        """Swap the table (train adj <-> test adj), as tf.assign does in supervised_train.py:260-261."""
        if adj_info.dtype != torch.int32 or adj_info.dim() != 2:
            raise TypeError("adj_info must be an int32 [N+1, max_degree] tensor")
        ops.require_cuda(adj_info)
        self.adj_info = adj_info.contiguous()

    def _call(self, inputs):
        ids, num_samples = inputs
        out = ops.sample_padded(self.adj_info, ids, int(num_samples), self.seed, self.counter,
                                counter_dev=self.counter_dev)
        self.counter += 1
        return out

    def sample_khop(self, ids, fanouts):
        """All hops of SampleAndAggregate.sample (reference models.py:254-275) in one kernel launch;
        identical to len(fanouts) successive calls.  fanouts in hop order, e.g. [10, 25]."""
        outs = ops.sample_padded_khop(self.adj_info, ids, [int(k) for k in fanouts], self.seed, self.counter,
                                      counter_dev=self.counter_dev)
        self.counter += len(fanouts)
        return outs


class CSRNeighborSampler(Layer):
    """Per-node uniform draws from a CSR adjacency (north_star's warp-per-node mode; the reference
    has only the padded table).  Same call convention as UniformNeighborSampler."""

    def __init__(self, indptr, indices, seed=123, replace_if_short=True, pad_id=None, **kwargs):
        super(CSRNeighborSampler, self).__init__(**kwargs)
        ops.require_cuda(indptr, indices)
        self.indptr, self.indices = indptr.contiguous(), indices.contiguous()
        self.seed = int(seed)
        self.counter = 0
        self.counter_dev = None
        self.replace_if_short = replace_if_short
        self.pad_id = int(indptr.numel() - 1) if pad_id is None else int(pad_id)   # dummy node N

    def _call(self, inputs):
        ids, num_samples = inputs
        out = ops.sample_csr(self.indptr, self.indices, ids, int(num_samples), self.seed, self.counter,
                             self.replace_if_short, self.pad_id, counter_dev=self.counter_dev)
        self.counter += 1
        return out


def _key(t):
    return (t.data_ptr(), t.numel(), t._version)


class WeightedNeighborSampler(Layer):
    """Fixed-fanout draws with replacement in proportion to a per-entry edge weight, from per-row alias tables
    (contract: oracle/alias_sampling.py).  Same call convention as UniformNeighborSampler: sampler((ids, k)) -> int32
    [n, k], sample_khop(ids, fanouts), `counter` (+1 per call, +len(fanouts) per sample_khop) and `counter_dev`, so
    SampleAndAggregate.sample, GraphedForward and graphed_train_step take it unchanged.  The sampled mean of k draws is
    an unbiased estimate of the w / sum(w) weighted mean of the row (PinSAGE-style importance sampling).

    indptr int64 [N + 1], indices int32 [E] and weights float32 [E] (one per entry; entries with finite w > 0 are drawn,
    a row with +inf entries draws uniformly among them, a row with none draws the dummy node N)."""

    def __init__(self, indptr, indices, weights, seed=123, **kwargs):
        super(WeightedNeighborSampler, self).__init__(**kwargs)
        self._tables = {}
        self.set_graph(indptr, indices, weights)
        self.seed = int(seed)
        self.counter = 0
        self.counter_dev = None   # optional device uint64 added to `counter` (CUDA-graph replay)

    def set_graph(self, indptr, indices, weights):
        """Swap the graph (train <-> test), the weighted counterpart of UniformNeighborSampler.set_adj.  The alias table
        of each graph is built once and kept, keyed by (data_ptr, numel, _version) of the three tensors, so swapping back
        does not rebuild, and a table a captured CUDA graph reads stays alive.  Every table is kept while the sampler
        lives, and a table takes 16 bytes per CSR entry (1.8 GB at Reddit's 114 M entries): changing a tensor in place
        (a new _version) builds and keeps another table, so update weights by building a new sampler, or expect one
        table per version.  A captured runner (GraphedForward, graphed_train_step) keeps drawing from the table it was
        captured with: capture a new one after a swap or a change of weights."""
        ops.require_cuda(indptr, indices)
        if indptr.dtype != torch.int64 or indptr.dim() != 1 or indptr.numel() < 1:
            raise TypeError("indptr must be a 1-D int64 tensor with >= 1 element")
        if indices.dtype != torch.int32 or indices.dim() != 1:
            raise TypeError("indices must be a 1-D int32 tensor")
        key = (_key(indptr), _key(indices), _key(weights) if isinstance(weights, torch.Tensor) else None)
        table = self._tables.get(key)
        if table is None:
            indptr, indices = indptr.contiguous(), indices.contiguous()
            table = (indptr, indices, weights, ops.csr_alias_table(indptr, indices, weights))
            self._tables[key] = table
        self.indptr, self.indices, self.weights, self.table = table

    def _call(self, inputs):
        ids, num_samples = inputs
        out = ops.sample_alias(self.indptr, self.table, ids, int(num_samples), self.seed, self.counter,
                               counter_dev=self.counter_dev)
        self.counter += 1
        return out

    def sample_khop(self, ids, fanouts):
        """All hops of SampleAndAggregate.sample in one kernel launch; identical to len(fanouts) successive calls.
        fanouts in hop order, e.g. [10, 25]."""
        outs = ops.sample_alias_khop(self.indptr, self.table, ids, [int(k) for k in fanouts], self.seed, self.counter,
                                     counter_dev=self.counter_dev)
        self.counter += len(fanouts)
        return outs
