"""Oracle for the Node2Vec / DeepWalk baseline (reference graphsage/models.py:408-501, Node2VecModel).

Unique unigram negatives - tf.nn.fixed_unigram_candidate_sampler(unique=True, distortion=0.75, unigrams=degrees)
(models.py:450-457).  TF draws candidates in sequence and rejects ids it already holds until it has num_sampled distinct
ids; the true classes do not change which ids are drawn.  TF's stream is unobtainable, so the raw draws follow the Philox
contract of oracle/sampler.py:sample_unigram on their own stream tag:
    draw j (j = 0, 1, ...) = word j&3 of philox4x32_10(ctr=(counter_lo, counter_hi, 0, UNIQUE tag + j>>2), key=seed)
    u = (draw + 0.5) / 2^32 * total;  id = first index whose inclusive float64 prefix sum exceeds u
and the result is the first num_sampled distinct ids of that sequence, in draw order.  After DRAW_BUDGET draws the
sampler gives up (the kernel writes -1 for the missing ids and raises a status flag).

Skip-gram step (models.py:459-486) with B = len(batch1), S = len(neg):
    t = T[batch1], c = C[batch2], cb = b[batch2], n = C[neg], nb = b[neg]
    aff = rowdot(t, c) (+ cb in the loss only), neg_aff = t n^T (+ nb in the loss only)
    loss = (sum softplus(-(aff + cb)) + sum softplus(neg_aff + nb)) / B
MRR (models.py:489-501): the bias-free affinities, columns [neg..., true], the two-top_k rank rule.
Update: plain gradient descent on the sparse gradient, duplicate ids summed (scatter_sub), every gradient taken from
the tables before the update.

Test infrastructure - not imported by the product.
"""
import numpy as np

from .sampler import _draws

STREAM_UNIGRAM_UNIQUE = 0x30000000
MAX_UNIQUE_SAMPLED = 1024
DRAW_BUDGET = 1 << 20


def unigram_cdf(degrees, distortion=0.75):
    return np.cumsum(np.asarray(degrees, dtype=np.float64) ** distortion)


def unique_support(degrees, distortion=0.75):
    """Number of ids with positive weight: the most distinct ids the sampler can return."""
    return int(np.count_nonzero(np.asarray(degrees, dtype=np.float64) ** distortion > 0))


def raw_unigram_draws(cdf, seed, counter, start, count):
    """Ids of draws start .. start + count - 1 of the unique sampler's stream."""
    assert start % 4 == 0
    r = _draws(seed, counter, count, c2=0, tag=STREAM_UNIGRAM_UNIQUE + start // 4).astype(np.float64)
    u = (r + 0.5) * (1.0 / 4294967296.0) * cdf[-1]
    return np.searchsorted(cdf, u, side="right").astype(np.int32)


def sample_unigram_unique(degrees, num_sampled, seed, counter, distortion=0.75, budget=DRAW_BUDGET):
    """The literal sequential rejection loop over the raw draws.  Returns int32[num_sampled] (-1 where the budget ran out)."""
    if num_sampled > MAX_UNIQUE_SAMPLED:
        raise ValueError("num_sampled > %d" % MAX_UNIQUE_SAMPLED)
    if num_sampled > unique_support(degrees, distortion):
        raise ValueError("num_sampled=%d exceeds the %d ids with positive weight" % (num_sampled,
                                                                                   unique_support(degrees, distortion)))
    cdf = unigram_cdf(degrees, distortion)
    out, held, j = [], set(), 0
    while len(out) < num_sampled and j < budget:
        block = raw_unigram_draws(cdf, seed, counter, j, min(1024, budget - j))
        for x in block:
            j += 1
            if int(x) not in held:
                held.add(int(x))
                out.append(int(x))
                if len(out) == num_sampled:
                    break
    return np.array(out + [-1] * (num_sampled - len(out)), dtype=np.int32)


def sample_unigram_unique_rounds(degrees, num_sampled, seed, counter, distortion=0.75, budget=DRAW_BUDGET):
    """The kernel's form of the same rule: rounds of 32 draws; a draw is accepted iff its id is neither held nor held by a
    lower draw of its round; accepted draws keep their order and the round is cut at num_sampled."""
    cdf = unigram_cdf(degrees, distortion)
    out, j0 = [], 0
    while len(out) < num_sampled and j0 < budget:
        ids = raw_unigram_draws(cdf, seed, counter, j0, min(32, budget - j0))
        for lane, x in enumerate(ids):
            if int(x) not in out and int(x) not in [int(y) for y in ids[:lane]] and len(out) < num_sampled:
                out.append(int(x))
        j0 += 32
    return np.array(out + [-1] * (num_sampled - len(out)), dtype=np.int32)


def _softplus(x):
    return np.maximum(x, 0) + np.log1p(np.exp(-np.abs(x)))


def _sigmoid(x):
    return 1.0 / (1.0 + np.exp(-x))


def skipgram_forward(T, C, b, batch1, batch2, neg):
    """(loss, aff, neg_aff) in float64; aff / neg_aff without the biases (what MRR ranks)."""
    T, C, b = (np.asarray(x, dtype=np.float64) for x in (T, C, b))
    t, c, n = T[batch1], C[batch2], C[neg]
    aff = (t * c).sum(1)
    neg_aff = t @ n.T
    B = len(batch1)
    loss = (_softplus(-(aff + b[batch2])).sum() + _softplus(neg_aff + b[neg][None, :]).sum()) / B
    return loss, aff, neg_aff


def skipgram_grads(T, C, b, batch1, batch2, neg):
    """Per-lookup gradients of the loss (float64): gt [B, d], gc_pos [B, d], gb_pos [B], gc_neg [S, d], gb_neg [S]."""
    T, C, b = (np.asarray(x, dtype=np.float64) for x in (T, C, b))
    t, c, n = T[batch1], C[batch2], C[neg]
    B = len(batch1)
    g = (_sigmoid((t * c).sum(1) + b[batch2]) - 1.0) / B               # d loss / d (aff_i + cb_i)
    h = _sigmoid(t @ n.T + b[neg][None, :]) / B                        # d loss / d (neg_aff_ij + nb_j)
    return dict(gt=g[:, None] * c + h @ n, gc_pos=g[:, None] * t, gb_pos=g, gc_neg=h.T @ t, gb_neg=h.sum(0))


def sgd_step(T, C, b, batch1, batch2, neg, lr):
    """One GradientDescentOptimizer(lr) step: the sparse gradients with duplicate ids summed (also across batch2 and the
    negatives), every gradient from the tables before the update.  Returns new float64 (T, C, b) and the loss."""
    loss, _, _ = skipgram_forward(T, C, b, batch1, batch2, neg)
    g = skipgram_grads(T, C, b, batch1, batch2, neg)
    T, C, b = (np.array(x, dtype=np.float64) for x in (T, C, b))
    np.subtract.at(T, np.asarray(batch1), lr * g["gt"])
    np.subtract.at(C, np.asarray(batch2), lr * g["gc_pos"])
    np.subtract.at(C, np.asarray(neg), lr * g["gc_neg"])
    np.subtract.at(b, np.asarray(batch2), lr * g["gb_pos"])
    np.subtract.at(b, np.asarray(neg), lr * g["gb_neg"])
    return T, C, b, loss


def ranks(aff, neg_aff):
    """models.py:496-500: the rank of every column of [neg..., true] by the two top_k passes (descending, ties to the
    lower column), and the MRR of the last column."""
    table = np.concatenate([np.asarray(neg_aff), np.asarray(aff)[:, None]], axis=1)
    by_score = np.argsort(-table, axis=1, kind="stable")
    rank = np.argsort(by_score, axis=1, kind="stable")
    return rank, float(np.mean(1.0 / (rank[:, -1] + 1.0)))
