"""Unsupervised GraphSAGE head around the hot path (SURVEY section 8f row 2; reference
graphsage/models.py:332-405 `_build` / `_loss` / `_accuracy`, graphsage/prediction.py:68-110).

Three passes of the hot path share one set of aggregators (batch1, batch2, and neg_sample_size negatives drawn with
probability ~ degree^0.75 and shared by the whole batch); skip-gram style cross-entropy on the l2-normalised
outputs; MRR of the true pair among the negatives.  Forward through the library's CUDA kernels, backward as in
supervised_models.py.
"""
import numpy as np
import torch

from . import ops
from .graphed_training import GraphedTrainStep
from .host_features import HostFeatures
from .models import SampleAndAggregate
from .prediction import BipartiteEdgePredLayer, mrr_from_affinities
from .supervised_models import (aggregator_parameters, build_aggregators, check_full_neighbor_dropout, clipped_step,
                                differentiable_outputs, embedding_parameters, init_dropout, refuse_distributed_embeddings,
                                refuse_distributed_host_table, refuse_fused_pool, weight_decay_term)


class UnigramNegativeSampler(object):
    """tf.nn.fixed_unigram_candidate_sampler(unique=False, distortion=0.75, unigrams=degrees) -
    reference graphsage/models.py:336-343.  One Philox call counter per sampler object."""

    def __init__(self, degrees, distortion=0.75, seed=123, device="cuda"):
        w = np.asarray(degrees, dtype=np.float64) ** distortion
        self.cdf = torch.from_numpy(np.cumsum(w)).to(device)
        self.seed, self.counter, self.counter_dev = int(seed), 0, None

    def __call__(self, num_sampled):
        out = ops.sample_unigram(self.cdf, int(num_sampled), self.seed, self.counter, counter_dev=self.counter_dev)
        self.counter += 1
        return out


class UnsupervisedGraphsage(SampleAndAggregate):
    """reference graphsage/models.py:187-405 (SampleAndAggregate with its unsupervised `_build`)."""

    def __init__(self, placeholders, features, adj, degrees, layer_infos, concat=True, aggregator_type="mean",
                 model_size="small", identity_dim=0, neg_sample_size=20, neg_sample_weights=1.0, learning_rate=0.00001,
                 weight_decay=0.0, seed=123, device="cuda", distributed=False, group=None, dropout_seed=12345,
                 fused_pool=False, **kwargs):
        """dropout_seed: key of the training dropout masks (placeholders['dropout'] > 0); with distributed=True each rank
        uses dropout_seed + rank.  fused_pool: train the maxpool / meanpool branch through the fused bf16 kernels (see
        SupervisedGraphsage)."""
        refuse_distributed_embeddings(identity_dim, distributed)
        refuse_distributed_host_table(features, distributed)
        super(UnsupervisedGraphsage, self).__init__(placeholders, features, adj, degrees, layer_infos, concat=concat,
                                                    aggregator_type=aggregator_type, model_size=model_size,
                                                    identity_dim=identity_dim, device=device, **kwargs)
        if aggregator_type not in ("mean", "gcn", "maxpool", "meanpool", "twomaxpool", "seq"):
            raise NotImplementedError("training is implemented for the mean, gcn, maxpool, meanpool, twomaxpool and seq "
                                      "aggregators")
        init_dropout(self, dropout_seed, distributed, group)
        self.neg_sample_size, self.neg_sample_weights = int(neg_sample_size), float(neg_sample_weights)
        self.learning_rate, self.weight_decay = learning_rate, weight_decay
        self.neg_sampler = UnigramNegativeSampler(degrees, 0.75, seed, device)      # models.py:336-343
        self.aggregators = build_aggregators(self)
        self.fused_pool = bool(fused_pool)
        refuse_fused_pool(self)
        if self.fused_pool and isinstance(features, HostFeatures) and features.dtype == torch.bfloat16:
            # K4's backward reads the bf16 working set itself, and the negatives' pass restages it before the backward
            raise NotImplementedError("fused_pool=True in the unsupervised model with a bfloat16 host-memory "
                                      "(HostFeatures) table is not implemented")
        dim_mult = 2 if self.concat else 1
        self.link_pred_layer = BipartiteEdgePredLayer(dim_mult * self.dims[-1], dim_mult * self.dims[-1], placeholders,
                                                      neg_sample_weights=self.neg_sample_weights, bilinear_weights=False,
                                                      device=device, name="edge_predict")      # models.py:362-365
        self.distributed, self.group, self.last_allreduce_bytes = bool(distributed), group, 0
        if self.distributed:                                                         # every rank starts from rank 0's weights
            from .parallel import broadcast_parameters
            broadcast_parameters(self.parameters(), 0, group)
        for p in self.parameters():
            p.requires_grad_(True)
        self.optimizer = torch.optim.Adam(self.parameters(), lr=self.learning_rate)

    def parameters(self):
        return aggregator_parameters(self.aggregators)[0] + embedding_parameters(self)

    def decayed_parameters(self):
        return aggregator_parameters(self.aggregators)[1]

    def embed(self, batch, dropout=0.):
        """dropout: the training rate (0 = the reference's evaluation default); each call draws fresh sites."""
        return differentiable_outputs(self, batch, dropout=dropout)                  # models.py:347-370

    def _passes(self, batch1, batch2, dropout=0.):
        neg = self.neg_sampler(self.neg_sample_size)
        o1, o2 = self.embed(batch1, dropout), self.embed(batch2, dropout)
        on = self.embed(neg, dropout)                                                # batch_size = neg_sample_size (:356-360)
        return o1, o2, on, neg

    def loss(self, batch1, batch2, dropout=0.):
        """weight decay + BipartiteEdgePredLayer._xent_loss (prediction.py:102-110), divided by the batch size
        (models.py:378).  The edge-prediction layer has no dropout (models.py:363-366)."""
        # at dropout 0 the two-argument form, which overrides of _passes implement
        o1, o2, on, _ = self._passes(batch1, batch2, dropout) if dropout else self._passes(batch1, batch2)
        return self._pairs_loss(o1, o2, on)

    def _pairs_loss(self, o1, o2, on):
        """loss()'s tail on the three passes' outputs, shared with full_neighbor_minibatch_loss; keeps the affinities
        for mrr()."""
        loss = self.link_pred_layer.loss(o1, o2, on)
        if self.weight_decay:
            loss = loss + weight_decay_term(self.decayed_parameters(), self.weight_decay)       # models.py:385-387
        with torch.no_grad():
            self._last = (self.link_pred_layer.affinity(o1, o2), self.link_pred_layer.neg_cost(o1, on))
        return loss / float(o1.shape[0])

    def mrr(self):
        """models.py:393-405 on the affinities of the last loss() call."""
        return mrr_from_affinities(*self._last)

    def train_step(self, batch1, batch2):
        return clipped_step(self, self.loss(batch1, batch2, dropout=self.dropout_rate))   # unsupervised_train.py:269

    def full_neighbor_minibatch_loss(self, indptr, indices, batch1, batch2, dropout=None, edge_weight=None):
        """loss() with every embedding computed over whole neighbourhoods (contract: oracle/full_neighbor_blocks.py): the
        negatives are drawn first, as _passes draws them (one neg_sampler call); ONE set of receptive-field blocks is
        built over cat(batch1, batch2, negatives) and its outputs split; then the same link-prediction loss and weight
        decay, divided by len(batch1), and the affinities for mrr().  Reads the block sizes back once per call.
        dropout: None, or a rate p in [0, 1) masking that one block set (SupervisedGraphsage.full_neighbor_outputs; there
        is no head site).  Refused (NotImplementedError): the seq aggregator, ShardedFeatures, distributed=True,
        CUDA-graph capture, and dropout=None on a model whose dropout_rate > 0.  edge_weight: the CSR's per-entry weights
        (SupervisedGraphsage.full_neighbor_outputs), refused with dropout p > 0."""
        from .full_neighbor_training import full_neighbor_outputs, refuse_full_neighbor, refuse_weighted_dropout
        check_full_neighbor_dropout(dropout)
        refuse_full_neighbor(self, training=True, dropout=dropout)                  # before drawing the negatives
        refuse_weighted_dropout(edge_weight, dropout)
        neg = self.neg_sampler(self.neg_sample_size)
        b1, b2 = (torch.as_tensor(b).to(device=self.device, dtype=torch.int32).reshape(-1) for b in (batch1, batch2))
        out = full_neighbor_outputs(self, indptr, indices, torch.cat([b1, b2, neg]), minibatch=True, dropout=dropout,
                                    edge_weight=edge_weight)
        return self._pairs_loss(*torch.split(out, [b1.numel(), b2.numel(), neg.numel()]))

    def full_neighbor_minibatch_train_step(self, indptr, indices, batch1, batch2, dropout=None, edge_weight=None):
        """One Adam step on full_neighbor_minibatch_loss, gradients clipped to +-5 as in train_step.  Returns the
        detached loss."""
        return clipped_step(self, self.full_neighbor_minibatch_loss(indptr, indices, batch1, batch2, dropout=dropout,
                                                                    edge_weight=edge_weight))

    def sampled_minibatch_loss(self, indptr, indices, batch1, batch2, dropout=None, edge_weight=None,
                               sample_weight=None):
        """loss() with every embedding computed over sampled receptive-field blocks (contract: oracle/sampled_blocks.py):
        the negatives are drawn first (one neg_sampler call), then ONE sampled block set over cat(batch1, batch2,
        negatives) - the sampler's counter advances by 1 - and its outputs split; then the same link-prediction loss and
        weight decay, divided by len(batch1), and the affinities for mrr().  dropout: None, or a rate p in [0, 1) masking
        that one block set (SupervisedGraphsage.sampled_minibatch_outputs; there is no head site).  Refusals as
        SupervisedGraphsage.sampled_minibatch_outputs, checked before the negatives are drawn.  edge_weight: as
        full_neighbor_minibatch_loss.  sample_weight: as SupervisedGraphsage.sampled_minibatch_outputs (the block set
        is drawn in proportion to it; the negatives stay the unigram draws)."""
        from .full_neighbor_training import full_neighbor_outputs, refuse_sampled, refuse_weighted_dropout
        check_full_neighbor_dropout(dropout)
        refuse_sampled(self, training=True, dropout=dropout)                        # before drawing the negatives
        refuse_weighted_dropout(edge_weight, dropout)
        neg = self.neg_sampler(self.neg_sample_size)
        b1, b2 = (torch.as_tensor(b).to(device=self.device, dtype=torch.int32).reshape(-1) for b in (batch1, batch2))
        out = full_neighbor_outputs(self, indptr, indices, torch.cat([b1, b2, neg]), minibatch=True, sampled=True,
                                    dropout=dropout, edge_weight=edge_weight, sample_weight=sample_weight)
        return self._pairs_loss(*torch.split(out, [b1.numel(), b2.numel(), neg.numel()]))

    def sampled_minibatch_train_step(self, indptr, indices, batch1, batch2, dropout=None, edge_weight=None,
                                     sample_weight=None):
        """One Adam step on sampled_minibatch_loss, gradients clipped to +-5 as in train_step.  Returns the detached
        loss."""
        return clipped_step(self, self.sampled_minibatch_loss(indptr, indices, batch1, batch2, dropout=dropout,
                                                              edge_weight=edge_weight, sample_weight=sample_weight))

    def graphed_train_step(self, batch_size):
        """train_step for a fixed batch size captured in one CUDA graph: returns step(batch1, batch2) -> loss, a static 0-d
        CUDA tensor (see graphed_training.GraphedTrainStep; a short last batch runs through the eager train_step)."""
        return GraphedTrainStep(self, batch_size)
