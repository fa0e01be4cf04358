"""Dropout masks for training: the counter-based contract shared by the CUDA kernels (graphsage_b200/csrc/common.cuh,
include/graphsage_b200.h: gs_dropout_site) and this oracle.

TensorFlow's tf.nn.dropout (reference aggregators.py:46-47, 104-105; layers.py:107) draws its mask from a stream that
cannot be reproduced without TensorFlow, like tf.random_shuffle (oracle/philox.py): "parity unpinned" for the stream,
pinned for everything computed from it - which tensors are dropped, in which order, and the x / keep_prob * mask scaling.

A SITE is one dropout application over a logical [rows, F] tensor, named by (seed, call), with rate p in [0, 1):
  element (pos, c) is kept iff word c % 4 of philox4x32_10(ctr = (c // 4, pos_lo32, pos_hi32, call), key = split64(seed))
  is >= T = floor(p * 2^32) (float64 arithmetic on the fp32 rate); a kept element becomes x / keep, keep = fp32(1 - p)
  (one IEEE fp32 division), a dropped element 0.
Positions: neighbour j of row i of an [n, k, F] neighbour tensor: pos = i * k + j; self rows: pos = i; a pooling MLP input
[n * k, F]: pos = row; the supervised head input: pos = batch row.  Columns are logical, 0 .. F - 1.

Test infrastructure - not imported by the product.
"""
import numpy as np

from .philox import philox4x32_10, split64

_ROWS_PER_CHUNK = 8192


def threshold(rate):
    """T = floor(p * 2^32) for the fp32 rate p."""
    p = np.float64(np.float32(rate))
    if not 0.0 <= p < 1.0:
        raise ValueError("dropout rate must be in [0, 1)")
    return np.uint32(int(np.floor(p * 4294967296.0)))


def keep_prob(rate):
    """keep = fp32(1 - p)."""
    return np.float32(1.0 - np.float64(np.float32(rate)))


def keep_mask(seed, call, rate, pos, F):
    """bool [len(pos), F]: True where element (pos[r], c) is kept."""
    pos = np.asarray(pos, dtype=np.int64).reshape(-1)
    T = threshold(rate)
    k0, k1 = split64(seed)
    key = np.array([k0, k1], dtype=np.uint32)
    n4 = (int(F) + 3) // 4
    out = np.empty((pos.size, n4 * 4), dtype=bool)
    c4 = np.arange(n4, dtype=np.uint64)
    for r0 in range(0, pos.size, _ROWS_PER_CHUNK):
        p = pos[r0:r0 + _ROWS_PER_CHUNK].astype(np.uint64)
        ctr = np.empty((p.size, n4, 4), dtype=np.uint32)
        ctr[..., 0] = c4[None, :].astype(np.uint32)
        ctr[..., 1] = (p & np.uint64(0xFFFFFFFF)).astype(np.uint32)[:, None]
        ctr[..., 2] = (p >> np.uint64(32)).astype(np.uint32)[:, None]
        ctr[..., 3] = np.uint32(int(call) & 0xFFFFFFFF)
        words = philox4x32_10(ctr, key)                              # [rows, n4, 4]: word e is column 4 * c4 + e
        out[r0:r0 + p.size] = (words >= T).reshape(p.size, n4 * 4)
    return out[:, :F]


def apply(x, seed, call, rate, pos=None):
    """drop(x) for x [rows, F] (pos defaults to the row index): where(mask, x / keep, 0) in fp32."""
    x = np.asarray(x, dtype=np.float32)
    rows, F = x.shape
    pos = np.arange(rows) if pos is None else pos
    m = keep_mask(seed, call, rate, pos, F)
    return np.where(m, x / keep_prob(rate), np.float32(0)).astype(np.float32)


def apply_nd(x, seed, call, rate):
    """drop(x) for a tensor of any rank: rows are the row-major flattening of every axis but the last (so an [n, k, F]
    neighbour tensor gets pos = i * k + j)."""
    x = np.asarray(x, dtype=np.float32)
    return apply(x.reshape(-1, x.shape[-1]), seed, call, rate).reshape(x.shape)


def aggregate_khop(samples, features, num_samples, support_sizes, batch_size, aggregators, concat, kind, rate, seed,
                   call0):
    """reference graphsage/models.py:278-330 with training dropout at `rate`, every site drawn in the reference's call
    order from call0 on: per layer, per hop, the neighbour then the self tensor (mean, gcn) or the MLP input (pools).
    aggregators: one dict per layer (oracle/aggregate.py names).  Returns (hidden[0], next call)."""
    from .aggregate import gather_rows, identity, relu
    call = call0
    hidden = [gather_rows(features, s).astype(np.float32) for s in samples]
    L = len(num_samples)
    for layer in range(L):
        act = identity if layer == L - 1 else relu
        w = aggregators[layer]
        nxt = []
        for hop in range(L - layer):
            F = hidden[hop + 1].shape[1]
            k = num_samples[L - hop - 1]
            neigh = hidden[hop + 1].reshape(batch_size * support_sizes[hop], k, F)
            selfv = hidden[hop]
            if kind in ("mean", "gcn"):
                neigh = apply_nd(neigh, seed, call, rate)
                selfv = apply(selfv, seed, call + 1, rate)
                call += 2
                if kind == "mean":
                    m = _mean_j(neigh)
                    fs, fn = selfv @ w["self_weights"], m @ w["neigh_weights"]
                    out = np.concatenate([fs, fn], axis=1) if concat else fs + fn
                else:
                    m = _mean_j(np.concatenate([neigh, selfv[:, None, :]], axis=1))
                    out = m @ w["weights"]
            else:
                n = neigh.shape[0]
                x = apply(neigh.reshape(n * k, F), seed, call, rate)
                call += 1
                h = relu(x @ w["mlp_weights"] + w["mlp_bias"]).reshape(n, k, -1)
                hp = h.max(axis=1) if kind == "maxpool" else _mean_j(h)
                fs, fn = selfv @ w["self_weights"], hp @ w["neigh_weights"]
                out = np.concatenate([fs, fn], axis=1) if concat else fs + fn
            nxt.append(act(out).astype(np.float32))
        hidden = nxt
    return hidden[0], call


def _mean_j(x):
    """mean over axis 1, summed in j order in fp32 (the gather kernels' order)."""
    acc = np.zeros((x.shape[0], x.shape[2]), dtype=np.float32)
    for j in range(x.shape[1]):
        acc += x[:, j]
    return acc / np.float32(x.shape[1])
