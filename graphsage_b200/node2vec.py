"""Node2Vec / DeepWalk baseline (reference graphsage/models.py:408-501, `Node2VecModel`; built by
graphsage/unsupervised_train.py:227-232): a target and a context embedding table trained by skip-gram with unique
unigram negatives and plain sparse gradient descent.  The hot path is three library calls per step, in a fixed order and
without host synchronisation:

    gs_sample_unigram_unique  S distinct negatives (tf.nn.fixed_unigram_candidate_sampler(unique=True), :450-457)
    gs_skipgram_grad          loss, affinities and the gradient of every lookup, from the tables before the update
    gs_embedding_sgd  x 2     target rows, then context rows + biases: table[r] -= lr * (summed gradient), touched rows only

The context bias is column d of the context table, so one sparse update covers both (`context_embeds` / `context_bias`
are views).  TF's random streams cannot be reproduced: the initialisers use a seeded torch generator, the sampler the
Philox contract of oracle/node2vec.py.
"""
import math

import numpy as np
import torch

from . import ops
from ._lib import MAX_UNIQUE_SAMPLED
from .graphed_training import GraphedTrainStep
from .prediction import mrr_from_affinities


def unique_support(degrees, distortion=0.75):
    """Number of ids with positive unigram weight: the most distinct negatives there are."""
    return int(np.count_nonzero(np.asarray(degrees, dtype=np.float64) ** distortion > 0))


def check_unique_sample_size(degrees, num_sampled, distortion=0.75):
    """ValueError unless num_sampled distinct ids can be drawn (TF's unique sampler would loop forever)."""
    num_sampled = int(num_sampled)
    if not 1 <= num_sampled <= MAX_UNIQUE_SAMPLED:
        raise ValueError("neg_sample_size must be in [1, %d] (got %d)" % (MAX_UNIQUE_SAMPLED, num_sampled))
    support = unique_support(degrees, distortion)
    if num_sampled > support:
        raise ValueError("neg_sample_size=%d distinct negatives requested, but only %d ids have a positive degree"
                         % (num_sampled, support))


class UniqueUnigramSampler(object):
    """tf.nn.fixed_unigram_candidate_sampler(unique=True, distortion=0.75, unigrams=degrees) - reference
    graphsage/models.py:450-457.  One Philox call counter per sampler object; each call draws fresh negatives.
    `status` (int32 CUDA [1]) turns 1 if a call ever ran out of its draw budget (see check())."""

    def __init__(self, degrees, num_sampled, distortion=0.75, seed=123, device="cuda"):
        check_unique_sample_size(degrees, num_sampled, distortion)
        w = np.asarray(degrees, dtype=np.float64) ** distortion
        self.num_sampled = int(num_sampled)
        self.cdf = torch.from_numpy(np.cumsum(w)).to(device)
        self.status = torch.zeros((1,), dtype=torch.int32, device=device)
        self.seed, self.counter, self.counter_dev = int(seed), 0, None

    def __call__(self):
        out = ops.sample_unigram_unique(self.cdf, self.num_sampled, self.seed, self.counter, counter_dev=self.counter_dev,
                                        status=self.status)
        self.counter += 1
        return out

    def check(self):
        """Raise if any call so far ran out of draws (synchronises with the device)."""
        if int(self.status.item()) != 0:
            raise RuntimeError("the unique unigram sampler ran out of its draw budget: the weights are too concentrated "
                               "for %d distinct ids" % self.num_sampled)


class Node2VecModel(object):
    """reference graphsage/models.py:408-501.  TF placeholders / FLAGS become arguments: `placeholders` is a plain dict
    (only read for compatibility), `neg_sample_size` is FLAGS.neg_sample_size, `seed` keys the initialisers and the
    negative sampler.  dict_size = V table rows (the trainer passes features.shape[0] = N + 1); degrees: the unigram
    counts of ids 0 .. len(degrees) - 1, the only ids drawn as negatives (the trainer passes the N train degrees)."""

    def __init__(self, placeholders, dict_size, degrees, name=None, nodevec_dim=50, lr=0.001, neg_sample_size=20, seed=123,
                 device="cuda"):
        V, d = int(dict_size), int(nodevec_dim)
        if V < 1 or d < 1:
            raise ValueError("dict_size and nodevec_dim must be >= 1")
        if len(degrees) > V:                  # negatives are ids < len(degrees) (range_max); the trainer passes N of N + 1
            raise ValueError("degrees has %d entries, more than dict_size = %d" % (len(degrees), V))
        check_unique_sample_size(degrees, neg_sample_size)                 # before any device work
        self.placeholders = placeholders if placeholders is not None else {}
        self.name = name or "node2vecmodel"
        self.degrees, self.hidden_dim, self.lr = degrees, d, float(lr)
        self.neg_sample_size = int(neg_sample_size)
        self.device = torch.device(device)
        gen = torch.Generator().manual_seed(int(seed))
        target = torch.empty((V, d), dtype=torch.float32).uniform_(-1.0, 1.0, generator=gen)      # tf.random_uniform(-1, 1)
        context = torch.empty((V, d), dtype=torch.float32)
        std = 1.0 / math.sqrt(d)                                           # tf.truncated_normal(stddev=1/sqrt(d))
        torch.nn.init.trunc_normal_(context, std=std, a=-2 * std, b=2 * std, generator=gen)
        self._target = torch.zeros((V, ops.pad_cols(d)), dtype=torch.float32, device=self.device)
        self._context = torch.zeros((V, ops.pad_cols(d + 1)), dtype=torch.float32, device=self.device)
        self._target[:, :d] = target.to(self.device)
        self._context[:, :d] = context.to(self.device)
        self.target_embeds = self._target[:, :d]
        self.context_embeds = self._context[:, :d]
        self.context_bias = self._context[:, d]                            # tf.zeros([dict_size])
        self.neg_sampler = UniqueUnigramSampler(degrees, self.neg_sample_size, 0.75, seed, self.device)
        self._last = None

    def _ids(self, x):
        return torch.as_tensor(x, dtype=torch.int32).reshape(-1).to(self.device, non_blocking=True)

    def _step(self, batch1, batch2):
        b1, b2 = self._ids(batch1), self._ids(batch2)
        neg = self.neg_sampler()
        out = ops.skipgram_grad(self.target_embeds, self._context[:, :self.hidden_dim + 1], b1, b2, neg)
        self._last = (out["aff"], out["neg_aff"])
        self.neg_samples = neg
        return b1, b2, neg, out

    def loss(self, batch1, batch2):
        """The loss of one batch on fresh negatives (models.py:478-486: softplus cross-entropies / B); no update."""
        return self._step(batch1, batch2)[3]["loss"]

    def train_step(self, batch1, batch2):
        """One sess.run of opt_op (unsupervised_train.py:269): fresh negatives, the gradients from the current tables,
        then the sparse gradient-descent updates of the target rows and of the context rows with their biases
        (duplicate ids summed, also across batch2 and the negatives).  Returns the loss (a 0-d CUDA tensor); no host sync."""
        b1, b2, neg, out = self._step(batch1, batch2)
        ops.embedding_sgd(self.target_embeds, [(b1, out["gt"], 1, 1.0)], self.lr)
        ops.embedding_sgd(self._context[:, :self.hidden_dim + 1], [(b2, out["gc_pos"], 1, 1.0), (neg, out["gc_neg"], 1, 1.0)],
                          self.lr)
        return out["loss"]

    def graphed_train_step(self, batch_size):
        """train_step for a fixed batch size captured in one CUDA graph: returns step(batch1, batch2) -> loss, a static 0-d
        CUDA tensor (see graphed_training.GraphedTrainStep; a short last batch runs through the eager train_step)."""
        return GraphedTrainStep(self, batch_size)

    def mrr(self):
        """models.py:489-501 on the bias-free affinities of the last loss() / train_step() call."""
        return mrr_from_affinities(*self._last)

    def outputs1(self, batch):
        """target_embeds[batch] (models.py:459): what save_val_embeddings exports."""
        return ops.gather_rows(self.target_embeds, self._ids(batch))

    def export_embeddings(self, node_ids, batch_size=512, out_prefix=None):
        """outputs1 of every given node (unsupervised_train.py:94-117), float32 [n, d]; with out_prefix also
        `<prefix>.npy` and `<prefix>.txt` (one id per line), the format of SampleAndAggregate.export_embeddings."""
        ids = torch.as_tensor(node_ids, dtype=torch.int32).reshape(-1)
        outs = [self.outputs1(ids[i:i + batch_size]).cpu() for i in range(0, ids.numel(), batch_size)]
        emb = torch.cat(outs).numpy() if outs else np.zeros((0, self.hidden_dim), np.float32)
        if out_prefix is not None:
            np.save(out_prefix + ".npy", emb)
            with open(out_prefix + ".txt", "w") as fp:
                fp.write("\n".join(str(int(x)) for x in ids.tolist()))
        return emb
