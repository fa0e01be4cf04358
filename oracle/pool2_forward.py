"""Operand-exact reference of K5's forward: gs_maxpool2_mlp_fused (csrc/maxpool2_tc.cu), the gather -> Dense(bias,
ReLU) -> Dense(bias, ReLU) -> max over each group's k rows of the bf16 two-layer max-pool aggregator, in one kernel.

Contract, for group g < n_groups and unit u of the second layer:

  operands  X[g, j] = the table row row(g, j), columns < K only, as stored in bf16 (widened exactly), addressed and
            clamped as in oracle/pool_forward.py.  W1 and W2 are rounded to bf16 to nearest even (maxpool_pack_kernel).
            Columns >= K and rows no group reads are never read.  A NULL bias is 0.
  pre1      the exact product X[g, j] . W1, accumulated in fp32 in an unspecified order.
  h1        bf16_rne(fmaxf(fl32(pre1 + b1), 0)).
  pre2_j    the exact product h1 . W2[:, u], accumulated the same way.
  out       fmaxf(fl32(max_j pre2_j) + b2[u], 0).

These are the operands of the materialised bf16 chain gs_gather_rows -> Dense (gs_sage_gemm, bias + ReLU) -> Dense ->
gs_segment_max: the bf16 GEMM rounds its A operand (the fp32 h1) to bf16 by RNE, and max commutes with the monotone
bias + ReLU.  K5 and the chain differ only in accumulation order.

Grid reference (grid_reference).  pool_forward's argument for layer 1: if S1 = sum_K |x w1| < 2^24 q(X) q(W1) and
S1 + |b1| < 2^24 min(q(X) q(W1), q(b1)), pre1 and pre1 + b1 are exact in fp32 whatever the order, so h1 is unique.
Then the same argument for layer 2 with X := h1, its quantum computed from the rounded h1 (pool_forward.grid_reference
asserts it).  Both sets of conditions are asserted from the operands; a test cannot pick ranges that silently round.

The aggregator itself (aggregator, aggregate_khop) is restated in numpy fp32 from the reference's op sequence, checked
against the reference's own class in tests/golden/twomax.npz.

Bounded reference (bounded_reference) for operands off the grid.
  layer 1  e1 = K 2^-23 S1_1 bounds the accumulated p1 against pre1 (numerics.gemm_bound's accumulation term, any order).
           With z = pre1 + b1 (exact) and t = e1 + ulp32(|z| + e1) (the fp32 rounding of p1 + b1), the kernel's fp32
           value v' = relu(fl32(p1 + b1)) lies in [relu(z - t), relu(z + t)], and so does the reference's v (p1 = pre1).
           v' is an fp32 number, so it also lies between the fp32 RNE roundings of the two ends, and RNE to bf16 is
           monotone: h1' = bf16_rne(v') and h1r = bf16_rne(v) both lie in [lo, hi] = the bf16 roundings of those ends.
             |h1' - h1r| <= dh1 = hi - lo.
           An accumulation error can flip the bf16 rounding by one step at most, and only where a rounding boundary lies
           within t of z: elsewhere dh1 = 0 and h1' = h1r exactly.  (The looser dh1 <= e1 + ulp_bf16(|h1| + e1) holds
           too; the interval form is tighter, so the checks see more.)
  layer 2  with pre2r = h1r . W2 (exact), the kernel's accumulated p2 satisfies
             |p2 - pre2r| <= |p2 - h1' . W2| + |(h1' - h1r) . W2| <= e2 = h1_w 2^-23 (|h1r| + dh1) . |W2| + dh1 . |W2|,
           h1_w the width of h1: K4's max bound (pool_forward's docstring) with the propagated layer-1 error added.
           E = max_j e2_j, ref = relu(max_j pre2r_j + b2): |out - ref| <= E + ulp32(ref + E).
  RMS      criterion (b) with pool_forward's subtraction: sqrt(mean((max(|out - ref| - R, 0) / S2*)^2)) <=
           numerics.RMS_BOUND, S2* the S2 = sqrt((h1r^2) . (W2^2)) of the row that attains the max.  R is what remains
           with exact accumulators: ulp32(ref), plus max_j (dh1 . |W2|)_j - the flips a rounding boundary within t allows,
           which move pre2 by whole bf16 steps of single terms (far more than 2^-17 S2) however accurate the
           accumulation.  Everywhere else h1 must be the reference's bits, so an h1 truncated, kept in fp32 or rounded
           after a missing bias shows in the statistic.

Test infrastructure - not imported by the product.
"""
import math

import numpy as np
import torch

from . import pool_forward as pf

row_index, gather, same_values, check_bounded = pf.row_index, pf.gather, pf.same_values, pf.check_bounded


def _bf16(x):
    """fp64 tensor -> fp32 -> bfloat16 by RNE -> fp64 (torch's float -> bfloat16 cast rounds to nearest even)."""
    return x.float().to(torch.bfloat16).double()


def hidden1(X, W1, b1):
    """(h1 fp64 [rows, h1] = bf16_rne(relu(fl32(pre1 + b1))) with pre1 exact, pre1, S1 = |X| |W1|, b1 fp64)."""
    X, W1b, b = pf._operands(X, W1, b1)
    pre = X @ W1b
    return _bf16(torch.relu((pre + b).float().double())), pre, X.abs() @ W1b.abs(), b


def grid_reference(X, W1, b1, W2, b2, k):
    """The contract's one answer on grid operands (module docstring), float32 [n_groups, h2] on X's device.  Raises
    AssertionError when the operands do not make every fp32 operation of the contract exact."""
    X, W1b, b = pf._operands(X, W1, b1)
    pre, S1 = X @ W1b, X.abs() @ W1b.abs()
    px, pw = pf._quantum_exp(X), pf._quantum_exp(W1b)
    p_pre = None if px is None or pw is None else px + pw
    p = pf._min_exp(p_pre, pf._quantum_exp(b))
    lim = 2.0 ** (24 + p) if p is not None else math.inf
    if p_pre is not None:
        assert float(S1.max()) < 2.0 ** (24 + p_pre), "pre1 is not exact in fp32 in every order"
    assert float((S1 + b.abs()).max()) < lim, "pre1 + b1 is not exact in fp32"
    z = pre.float() + b.float()
    assert torch.equal(pre.float().double(), pre) and torch.equal(z.double(), pre + b)
    h1 = _bf16(torch.relu(z.double()))
    return pf.grid_reference(h1, W2, b2, k, "max")


def bounded_reference(X, W1, b1, W2, b2, k):
    """(ref, bound, s2, r): the fp64 contract output [n_groups, h2], the derived bound on |out - ref|, and the S2* and R
    of the RMS statistic (module docstring), all fp64 on X's device."""
    h1, pre1, S1, b = hidden1(X, W1, b1)
    K = pf._t(X).shape[1]
    z = pre1 + b
    e1 = (K * 2.0 ** -23) * S1
    t = e1 + pf._ulp32(z.abs() + e1)
    dh1 = _bf16(torch.relu(z + t)) - _bf16(torch.relu(z - t))
    _, W2b, b2 = pf._operands(h1, W2, b2)
    aW2 = W2b.abs()
    pre2 = h1 @ W2b
    flip = dh1 @ aW2
    e2 = (h1.shape[1] * 2.0 ** -23) * ((h1.abs() + dh1) @ aW2) + flip
    S2 = torch.sqrt((h1 * h1) @ (W2b * W2b))
    n, h2 = pre2.shape[0] // k, pre2.shape[1]
    r, arg = (pre2 + b2).reshape(n, k, h2).max(dim=1)
    ref = torch.relu(r)
    E = e2.reshape(n, k, h2).max(dim=1).values
    s2 = torch.gather(S2.reshape(n, k, h2), 1, arg[:, None, :])[:, 0]
    return ref, E + pf._ulp32(ref + E), s2, pf._ulp32(ref) + flip.reshape(n, k, h2).max(dim=1).values


def weights_from_draws(draws):
    """The reference aggregator's W1, W2, neigh_weights, self_weights from tests/golden/twomax.npz's (seed, rows, cols)
    records: U(-r, r), r = sqrt(6 / (rows + cols)), from numpy's RandomState(seed) (oracle.seq.cell_kernel)."""
    from .seq import cell_kernel
    names = ("W1", "W2", "neigh_weights", "self_weights")
    return {name: cell_kernel(int(s), (int(r), int(c))) for name, (s, r, c) in zip(names, np.asarray(draws))}


def aggregator(selfv, neigh, w, concat, relu_out=True, drop=None):
    """TwoMaxLayerPoolingAggregator._call (reference aggregators.py:330-361) in numpy fp32: each Dense (layers.py:104-116)
    is relu(drop(x) @ W + b) on the [n*k, .] rows, then the max over the k rows, the two products, concat or add, the
    optional bias, the activation.  w: W1, b1, W2, b2, neigh_weights, self_weights [, bias]; drop: None, or a callable
    applied to each Dense input in call order."""
    n, k, d = neigh.shape
    h = np.asarray(neigh, np.float32).reshape(n * k, d)
    for W, b in ((w["W1"], w["b1"]), (w["W2"], w["b2"])):
        if drop is not None:
            h = drop(h)
        h = np.maximum(h @ W + b, 0).astype(np.float32)
    hp = h.reshape(n, k, -1).max(axis=1)
    fs, fn = selfv @ w["self_weights"], hp @ w["neigh_weights"]
    out = np.concatenate([fs, fn], axis=1) if concat else fs + fn
    if "bias" in w:
        out = out + w["bias"]
    return (np.maximum(out, 0) if relu_out else out).astype(np.float32)


def aggregate_khop(samples, features, num_samples, support_sizes, batch_size, weights, concat, drop=None):
    """SampleAndAggregate.aggregate (reference models.py:278-330) with this aggregator: layer l calls aggregator() once
    per hop, the last layer without the ReLU."""
    L = len(num_samples)
    hidden = [np.asarray(features)[np.asarray(s).astype(np.int64)] for s in samples]
    for layer in range(L):
        nxt = []
        for hop in range(L - layer):
            neigh = hidden[hop + 1].reshape(batch_size * support_sizes[hop], num_samples[L - hop - 1], -1)
            nxt.append(aggregator(hidden[hop], neigh, weights[layer], concat, layer != L - 1, drop))
        hidden = nxt
    return hidden[0]


def full_neighbor_embeddings(features, indptr, indices, weights, concat, node_ids=None, normalize=True):
    """oracle/full_neighbor.py's layer loop with this aggregator's pooling branch: every node's two Dense layers once,
    relu(relu(h W1 + b1) W2 + b2), then the max over its CSR row (the dummy node N for an empty row), combined with the
    self rows as full_neighbor.layer does.  weights: one dict per layer as aggregator() takes.  numpy fp32."""
    from . import full_neighbor as fn
    h = np.asarray(features, dtype=np.float32)
    N = h.shape[0] - 1
    node_ids = np.arange(N) if node_ids is None else np.asarray(node_ids, dtype=np.int64).reshape(-1)
    L = len(weights)
    for layer, w in enumerate(weights):
        rows = node_ids if layer == L - 1 else None
        z = np.maximum(np.maximum(h @ w["W1"] + w["b1"], 0).astype(np.float32) @ w["W2"] + w["b2"], 0)
        p = fn.csr_aggregate(z.astype(np.float32), indptr, indices, "max", rows)
        hs = h if rows is None else fn.gather_clamped(h, rows)
        y = fn._combine(hs @ w["self_weights"], p @ w["neigh_weights"], concat)
        if "bias" in w:
            y = y + w["bias"]
        h = (y if layer == L - 1 else np.maximum(y, 0)).astype(np.float32)
    return fn.l2_normalize(h) if normalize else h
