"""Sampling neighbours in proportion to edge weight, without a GPU: neg_log against math.log, the weighted sample
contract (oracle/weighted_sampling.py) against a scalar restatement, eligibility, the law of the draws, the block
invariants, gradients through weighted blocks against float64 autograd, the autograd wiring of sample_weight= with the
oracle standing in for the kernels (TEST mocks only: the product has no such path), and the argument errors."""
import itertools
import math
import types

import numpy as np
import pytest
import torch

from graphsage_b200 import ops
from graphsage_b200.supervised_models import SupervisedGraphsage
from graphsage_b200.unsupervised_models import UnsupervisedGraphsage
from oracle import full_neighbor_blocks as fb
from oracle import sampled_blocks as sb
from oracle import weighted_sampling as ws
from oracle.philox import philox4x32_10, split64
from test_full_neighbor_minibatch_cpu import (_FakeNegatives, _cpu_model, _fake_csr_blocks, block_kernels,  # noqa: F401
                                              hub_graph)
from test_full_neighbor_train_cpu import CSR, _agg_dicts, _np, _torch_formula, cpu_kernels  # noqa: F401
from test_sampled_blocks_cpu import _sampled_bare, _with_sampler, fnt_oracle_dicts, rows_graph

NEG_LOG_ULP = 2


# ---------------------------------------------------------------- neg_log
def _ulps(u):
    got = ws.neg_log(u)
    ref = np.array([-math.log(x) for x in u])
    return np.abs(got - ref) / np.spacing(ref)


def test_neg_log_within_its_ulp_bound():
    ends = np.array([2.0 ** -53, 1 - 2.0 ** -53, 0.5, 0.5 + 2.0 ** -53, 1 / math.sqrt(2), math.sqrt(0.5) * 2 ** -9])
    assert _ulps(ends).max() <= NEG_LOG_ULP
    powers = np.array([2.0 ** -i for i in range(1, 54)])
    assert _ulps(powers).max() <= NEG_LOG_ULP
    m = np.random.RandomState(0).randint(0, 2 ** 52, size=10 ** 6, dtype=np.int64).astype(np.uint64)
    u = (2 * m + 1).astype(np.float64) * 2.0 ** -53
    assert _ulps(u).max() <= NEG_LOG_ULP


def test_neg_log_is_monotone():
    r = np.random.RandomState(1)
    m = np.unique(np.concatenate([r.randint(0, 2 ** 52, size=10 ** 6, dtype=np.int64),
                                  np.arange(2 ** 20), 2 ** 52 - 1 - np.arange(2 ** 20),
                                  (2 ** 51 + np.arange(-2 ** 16, 2 ** 16))])).astype(np.uint64)
    e = ws.neg_log((2 * m + 1).astype(np.float64) * 2.0 ** -53)
    assert np.all(np.diff(e) <= 0) and e.min() > 0


# ---------------------------------------------------------------- the sample
def scalar_sample(indptr, indices, w, v, k, seed, call, layer):
    """S_layer^w(v) one entry at a time, straight from the contract's words (Python floats: IEEE fp64 division)."""
    lo, hi = int(indptr[v]), int(indptr[v + 1])
    cand = []
    for j in range(max(hi - lo, 0)):
        wj = float(w[lo + j])
        if not wj > 0:
            continue
        ctr = np.array([j >> 1, v, call & 0xFFFFFFFF, 0x80000000 | layer], np.uint32)
        r = [int(x) for x in philox4x32_10(ctr, np.array(split64(seed), np.uint32))]
        a, b = (r[2], r[3]) if j & 1 else (r[0], r[1])
        m = (a << 20) | (b >> 12)
        e = float(ws.neg_log(np.array([(2 * m + 1) * 2.0 ** -53]))[0])
        key = e / wj if wj != math.inf else 0.0
        cand.append((key, j))
    chosen = sorted(j for _, j in sorted(cand)[:k])
    return [int(indices[lo + j]) for j in chosen], chosen


def weight_kinds(n, r):
    """Weights of several kinds, one per entry: positive, with zeros, negatives, NaN, +inf, subnormals, all equal."""
    pos = r.uniform(0.01, 5, n).astype(np.float32)
    mixed = pos.copy()
    sel = r.randint(0, 6, n)
    mixed[sel == 0] = 0
    mixed[sel == 1] = -1
    mixed[sel == 2] = np.nan
    mixed[sel == 3] = np.inf
    mixed[sel == 4] = np.float32(1e-40)
    return {"positive": pos, "mixed": mixed, "equal": np.full(n, 0.5, np.float32),
            "heavy": np.exp(r.randn(n) * 4).astype(np.float32)}


@pytest.mark.parametrize("k", [1, 3, 10, 25, 256])
def test_sample_rows_equal_the_scalar_restatement(k):
    degrees = [0, 1, k - 1 if k > 1 else 0, k, k + 1, 2 * k + 3, 600, 5, 0, 300]
    indptr, indices = rows_graph(degrees)
    r = np.random.RandomState(k)
    for name, w in weight_kinds(len(indices), r).items():
        for seed, call, layer in [(0, 0, 0), (123, 7, 1), (2 ** 63 + 5, 2 ** 40 + 3, 7)]:
            s_ptr, s_idx = ws.sample_rows(indptr, indices, w, k, seed, call, layer)
            o_ptr, offs = ws.sample_offsets(indptr, w, k, seed, call, layer)
            assert np.array_equal(s_ptr, o_ptr)
            for v in range(len(degrees)):
                want, pos = scalar_sample(indptr, indices, w, v, k, seed, call, layer)
                assert s_idx[s_ptr[v]:s_ptr[v + 1]].tolist() == want, (name, k, v, seed)
                assert offs[o_ptr[v]:o_ptr[v + 1]].tolist() == pos


def test_eligibility():
    indptr = np.array([0, 6, 10, 13, 13, 20], np.int64)
    indices = np.arange(20, dtype=np.int32) + 100
    w = np.array([0, -2, np.nan, 1, 0, 3,          # row 0: two eligible
                  np.inf, 1, np.inf, 2,            # row 1: the +inf entries come first
                  0, -0.0, np.nan,                 # row 2: none eligible
                  5, 1, 2, 0, 7, 9, 4], np.float32)
    ptr, idx = ws.sample_rows(indptr, indices, w, 2, 3, 1, 0)
    assert np.diff(ptr).tolist() == [2, 2, 0, 0, 2]
    assert idx[ptr[0]:ptr[1]].tolist() == [103, 105]                 # d+ <= k: every eligible entry, CSR order
    assert idx[ptr[1]:ptr[2]].tolist() == [106, 108]                 # key 0, ordered by position
    assert set(idx[ptr[4]:ptr[5]].tolist()) <= {113, 114, 115, 117, 118, 119}
    for seed in range(50):                                           # never a zero, negative or NaN weight
        _, idx = ws.sample_rows(indptr, indices, w, 1, seed, 0, 0)
        assert not set(idx.tolist()) & {100, 101, 102, 104, 110, 111, 112, 116}
    # an all-ineligible row is empty, and its block reads the dummy
    blocks = ws.sampled_blocks(indptr, indices, w, np.array([2]), [3], 0, 0)
    b = blocks[0]
    assert b["src_ids"].tolist() == [2, 5] and b["indptr"].tolist() == [0, 0] and b["rows"].tolist() == [0]


def test_words_layer_call_and_seed_select_other_samples():
    indptr, indices = rows_graph([60] * 8)
    w = np.random.RandomState(0).uniform(0.1, 1, len(indices)).astype(np.float32)
    base = ws.sample_rows(indptr, indices, w, 5, 1, 2, 3)[1]
    for other in [(1, 2, 4), (1, 3, 3), (2, 2, 3)]:
        assert not np.array_equal(base, ws.sample_rows(indptr, indices, w, 5, *other)[1])
    assert np.array_equal(base, ws.sample_rows(indptr, indices, w, 5, 1, 2 + 2 ** 32, 3)[1])   # call mod 2^32


# ---------------------------------------------------------------- the law
def _subset_probabilities(w, k):
    """The exact inclusion probability of every k-subset under successive sampling in proportion to w."""
    p = {}
    for seq in itertools.permutations(range(len(w)), k):
        left, q = float(sum(w)), 1.0
        for j in seq:
            q *= w[j] / left
            left -= w[j]
        key = frozenset(seq)
        p[key] = p.get(key, 0.0) + q
    return p


def _subset_counts(w, k, n, seed):
    d = len(w)
    indptr = np.arange(n + 1, dtype=np.int64) * d
    ptr, off = ws.sample_offsets(indptr, np.tile(np.asarray(w, np.float32), n), k, seed, 4, 1)
    assert np.all(np.diff(ptr) == k)
    code = (1 << off.reshape(n, k)).sum(axis=1)
    return np.bincount(code, minlength=1 << d)


@pytest.mark.parametrize("weights", [[1, 2, 3, 4, 5, 6], [0.5, 8, 1, 0.25, 3, 2], [1] * 6])
def test_inclusion_frequencies_follow_successive_sampling(weights):
    n, k = 200000, 3
    w = np.asarray(weights, np.float32).astype(np.float64)
    probs = _subset_probabilities(w, k)
    counts = _subset_counts(weights, k, n, 77)
    assert sum(counts[sum(1 << j for j in s)] for s in probs) == n
    for s, p in probs.items():
        c = counts[sum(1 << j for j in s)]
        assert abs(c - n * p) < 5 * np.sqrt(n * p * (1 - p)) + 1, (sorted(s), c, n * p)
    if len(set(weights)) == 1:
        assert all(abs(p - 1 / 20) < 1e-12 for p in probs.values())


# ---------------------------------------------------------------- the blocks
@pytest.mark.parametrize("L", [1, 2, 3])
@pytest.mark.parametrize("fan", [1, 3, 256])
def test_block_invariants(L, fan):
    indptr, indices = hub_graph(N=60, seed=L)
    N = len(indptr) - 1
    w = weight_kinds(len(indices), np.random.RandomState(L))["mixed"]
    fanouts = [fan, max(1, fan - 1), fan][:L]
    for seeds in (np.array([3, 3, -1, N, N + 5, 0, 17, 2]), np.arange(N), np.array([7]), np.zeros(0, np.int64)):
        blocks, offsets = ws.entry_offsets(indptr, indices, w, seeds, fanouts, 11, 4)
        nxt = fb.clamp_ids(seeds, N)
        for l in range(L - 1, -1, -1):
            b = blocks[l]
            V = b["src_ids"].astype(np.int64)
            members = set(np.unique(nxt).tolist())
            assert np.all(np.diff(V) > 0) and V[-1] == N
            assert set(nxt.tolist()) <= set(V.tolist()) and np.array_equal(V[b["rows"]], nxt)
            s_ptr, s_idx = ws.sample_rows(indptr, indices, w, fanouts[l], 11, 4, l)
            o_ptr, o = ws.sample_offsets(indptr, w, fanouts[l], 11, 4, l)
            for p, v in enumerate(V[:-1]):
                lo, hi = b["indptr"][p], b["indptr"][p + 1]
                want = fb.clamp_ids(s_idx[s_ptr[v]:s_ptr[v + 1]], N) if v in members else []
                assert np.array_equal(V[b["indices"][lo:hi]], want)
                if v in members:
                    assert np.array_equal(offsets[l][lo:hi], o[o_ptr[v]:o_ptr[v + 1]])
                    assert np.array_equal(indices[indptr[v] + offsets[l][lo:hi]], s_idx[s_ptr[v]:s_ptr[v + 1]])
            nxt = V


def test_large_fanouts_with_positive_weights_give_the_whole_neighbourhood_blocks():
    indptr, indices = hub_graph(N=60, seed=2)
    w = np.random.RandomState(3).uniform(0.01, 9, len(indices)).astype(np.float32)
    seeds = np.array([3, 3, -1, 60, 0, 17, 2])
    for L in (1, 2, 3):
        want = fb.csr_blocks(indptr, indices, seeds, L)
        got = ws.sampled_blocks(indptr, indices, w, seeds, [256] * L, 5, 9)
        for a, b in zip(got, want):
            for key in a:
                assert np.array_equal(a[key], b[key]) and a[key].dtype == b[key].dtype


@pytest.mark.parametrize("kind,concat,d", [("mean", True, 0), ("gcn", False, 16), ("maxpool", True, 16),
                                           ("meanpool", False, 0)])
def test_gradients_equal_float64_autograd_over_the_sample(kind, concat, d):
    r = np.random.RandomState(9)
    indptr, indices = hub_graph(N=30, seed=3)
    N, F, C = len(indptr) - 1, 5, 3
    w = weight_kinds(len(indices), r)["heavy"]
    x = r.randn(N + 1, F).astype(np.float32)
    x[N] = 0
    feats = np.concatenate([r.randn(N + 1, d).astype(np.float32), x], 1) if d else x
    aggs = _agg_dicts(kind, [d + F, 4], concat, r)
    node_ids = np.array([0, 3, 5, 5, 9, 2, 11, 29], np.int64)
    out_w = 4 * (2 if concat and kind != "gcn" else 1)
    pred_w, pred_b = (r.randn(out_w, C) * 0.5).astype(np.float32), (r.randn(C) * 0.1).astype(np.float32)
    labels = np.eye(C)[r.randint(0, C, len(node_ids))]
    loss, grads, head, demb = ws.loss_grads(feats, indptr, indices, w, aggs, concat, node_ids, labels, pred_w, pred_b,
                                            [2], 4, 0, False, 0.01, d)
    s_ptr, s_idx = ws.sample_rows(indptr, indices, w, 2, 4, 0, 0)
    rl, rgrads, rhead, rdemb = _torch_formula(feats, s_ptr, s_idx.astype(np.int32), aggs, concat, node_ids, pred_w,
                                              pred_b, labels, False, 0.01, d)
    assert abs(loss - rl) < 1e-5 * max(1, abs(rl))

    def close(a, b, what):
        assert a.shape == b.shape, what
        assert np.abs(a - b).max() <= 1e-4 * max(1.0, np.abs(b).max()), (what, np.abs(a - b).max())
    for g, rg in zip(grads, rgrads):
        for key in g:
            close(g[key], rg[key], key)
    close(head["weights"], rhead["weights"], "head")
    if d:
        close(demb, rdemb, "embeddings")


# ---------------------------------------------------------------- the autograd wiring, kernels replaced by the oracle
def _fake_weighted_blocks(indptr, indices, seeds, n_layers, fanouts=None, seed=0, call=0, entry_offsets=False,
                          sample_weights=None):
    assert fanouts is not None and sample_weights is not None and not entry_offsets
    return [ops.CsrBlock(*(torch.from_numpy(np.asarray(b[key])) for key in ("src_ids", "indptr", "indices", "rows")))
            for b in ws.sampled_blocks(_np(indptr), _np(indices), _np(sample_weights), _np(seeds), fanouts, seed, call)]


@pytest.fixture()
def weighted_kernels(block_kernels, monkeypatch):
    monkeypatch.setattr(ops, "csr_blocks", _fake_weighted_blocks)


@pytest.mark.parametrize("kind,concat,d", [("mean", True, 0), ("gcn", False, 16), ("maxpool", True, 16),
                                           ("meanpool", False, 0)])
def test_supervised_wiring_matches_the_weighted_oracle(weighted_kernels, kind, concat, d):
    model, indptr, indices = _cpu_model(SupervisedGraphsage, kind, concat, d)
    sampler = _with_sampler(model)
    r = np.random.RandomState(2)
    w = weight_kinds(len(indices), r)["mixed"]
    node_ids = np.array([1, 4, 4, 7, 2, 39, -3], np.int64)
    labels = np.eye(3)[r.randint(0, 3, len(node_ids))]
    loss = model.sampled_minibatch_loss(indptr, indices, node_ids, labels, sample_weight=w)
    assert sampler.counter == 4
    loss.backward()
    fanouts = [info.num_samples for info in model.layer_infos]
    rl, grads, head, demb = ws.loss_grads(_np(model.features), indptr, indices, w, fnt_oracle_dicts(model), concat,
                                          node_ids, labels, _np(model.node_pred_vars["weights"]),
                                          _np(model.node_pred_vars["bias"]), fanouts, 5, 3, False, 0.01, d)
    assert abs(float(loss.detach()) - rl) < 1e-5

    def close(t, ref, what):
        assert t.grad is not None, what
        assert np.abs(_np(t.grad) - ref).max() <= 1e-4 * max(1.0, np.abs(ref).max()), what
    for a, g in zip(model.aggregators, grads):
        for key, v in a.vars.items():
            close(v, g[key], key)
        if hasattr(a, "mlp_layers"):
            close(a.mlp_layers[0].vars["weights"], g["mlp_weights"], "mlp_weights")
    close(model.node_pred_vars["weights"], head["weights"], "head")
    if d:
        close(model.embeds, demb, "embeds")
    with torch.no_grad():
        emb = model.sampled_minibatch_embeddings(indptr, indices, node_ids, sample_weight=torch.from_numpy(w))
    want = ws.embeddings(_np(model.features), indptr, indices, w, fnt_oracle_dicts(model), concat, node_ids, fanouts,
                         5, 4)
    assert np.abs(_np(emb) - want).max() < 1e-5 and sampler.counter == 5
    before = [p.detach().clone() for p in model.parameters()]
    model.sampled_minibatch_train_step(indptr, indices, node_ids, labels, sample_weight=w)
    assert sampler.counter == 6
    assert any(not torch.equal(a, p.detach()) for a, p in zip(before, model.parameters()))


def test_unsupervised_wiring(weighted_kernels):
    from graphsage_b200 import full_neighbor_training as fnt
    model, indptr, indices = _cpu_model(UnsupervisedGraphsage, "mean", True, 0, neg_sample_size=4)
    sampler = _with_sampler(model, seed=9, counter=0)
    model.neg_sampler = _FakeNegatives([5, 0, 33, 5])
    w = weight_kinds(len(indices), np.random.RandomState(4))["heavy"]
    b1, b2 = np.array([1, 2, 3, 9]), np.array([4, 4, 38, 0])
    loss = model.sampled_minibatch_loss(indptr, indices, b1, b2, sample_weight=w)
    assert model.neg_sampler.counter == 1 and sampler.counter == 1
    loss.backward()
    sampler.counter = 0
    out = fnt.full_neighbor_outputs(model, indptr, indices, torch.cat([torch.tensor(b1), torch.tensor(b2),
                                                                       model.neg_sampler.ids.long()]),
                                    minibatch=True, sampled=True, sample_weight=w)
    assert torch.equal(loss.detach(), model._pairs_loss(*torch.split(out, [4, 4, 4])).detach())
    model.sampled_minibatch_train_step(indptr, indices, b1, b2, sample_weight=w)
    assert model.neg_sampler.counter == 2 and sampler.counter == 2


# ---------------------------------------------------------------- refusals and argument errors
def test_refusals_and_argument_errors(monkeypatch):
    w = np.ones(4, np.float32)
    with pytest.raises(NotImplementedError, match="seq"):
        _sampled_bare("seq").sampled_minibatch_train_step(*CSR, [0], [[1.0]], sample_weight=w)
    m = _sampled_bare()
    m.features = type("Sharded", (), {"c_table": lambda self: None, "shape": (5, 3)})()
    with pytest.raises(NotImplementedError, match="ShardedFeatures"):
        m.sampled_minibatch_loss(*CSR, [0], [[1.0]], sample_weight=w)
    m = _sampled_bare(aggregators=[])
    n = len(CSR[1])
    for bad, err, what in [(np.ones(n, np.float64), TypeError, "float32"), (torch.ones(n, dtype=torch.float64),
                           TypeError, "float32"), (np.ones(n + 1, np.float32), ValueError, "one weight per CSR entry"),
                           (torch.ones((n, 1)), ValueError, "one weight per CSR entry")]:
        with pytest.raises(err, match="sample_weight.*" + what):
            m.sampled_minibatch_embeddings(*CSR, [0], sample_weight=bad)
        assert m.layer_infos[0].neigh_sampler.counter == 0                # refused before any draw
    for name in ("full_neighbor_embeddings", "full_neighbor_minibatch_embeddings"):
        with pytest.raises(TypeError, match="sample_weight"):
            getattr(m, name)(*CSR, [0], sample_weight=w)
    monkeypatch.setattr(torch.cuda, "is_available", lambda: True)
    monkeypatch.setattr(torch.cuda, "is_current_stream_capturing", lambda: True)
    with pytest.raises(NotImplementedError, match="CUDA graph"):
        _sampled_bare().sampled_minibatch_train_step(*CSR, [0], [[1.0]], sample_weight=np.ones(n, np.float32))


def test_ops_check_their_arguments_and_have_no_cpu_fallback():
    indptr, indices = torch.zeros(3, dtype=torch.int64), torch.zeros(0, dtype=torch.int32)
    with pytest.raises(ValueError, match="sample_weights needs fanouts"):
        ops.csr_blocks(indptr, indices, torch.zeros(1, dtype=torch.int32), 2, sample_weights=torch.zeros(0))
    with pytest.raises(RuntimeError, match="CUDA-only"):
        ops.csr_blocks(indptr, indices, torch.zeros(1, dtype=torch.int32), 2, fanouts=[3, 3],
                       sample_weights=torch.zeros(0))
    with pytest.raises(RuntimeError, match="CUDA-only"):
        ops.sample_csr_rows(indptr, indices, 3, 0, 0, 0, weights=torch.zeros(0))
    with pytest.raises(ValueError, match="fanout"):
        ws.sample_rows(*rows_graph([3]), np.ones(3, np.float32), 257, 0, 0, 0)
    with pytest.raises(ValueError, match="float32"):
        ws.sample_rows(*rows_graph([3]), np.ones(3), 2, 0, 0, 0)
