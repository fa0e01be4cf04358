"""Minibatches over sampled neighbourhoods without a GPU: the sample contract (oracle/sampled_blocks.py) against a scalar
restatement of Floyd's algorithm, its edge cases, the block invariants, gradients through sampled blocks against float64
autograd of the whole-graph formula over the sample, the law of the draws, the autograd wiring of sampled_minibatch_*
with the oracle standing in for the kernels (TEST mocks only: the product has no such path), and the refusals."""
import types

import numpy as np
import pytest
import torch

from graphsage_b200 import full_neighbor_training as fnt
from graphsage_b200 import ops
from graphsage_b200.supervised_models import SupervisedGraphsage
from graphsage_b200.unsupervised_models import UnsupervisedGraphsage
from oracle import full_neighbor_blocks as fb
from oracle import sampled_blocks as sb
from oracle.philox import philox4x32_10, split64
from test_full_neighbor_minibatch_cpu import (_FakeNegatives, _cpu_model, _fake_csr_blocks, block_kernels,  # noqa: F401
                                              hub_graph)
from test_full_neighbor_train_cpu import CSR, _agg_dicts, _bare_model, _np, _torch_formula, cpu_kernels  # noqa: F401


def scalar_sample(indptr, indices, v, k, seed, call, layer):
    """S_layer(v) one move at a time, straight from the contract's words."""
    lo, hi = int(indptr[v]), int(indptr[v + 1])
    d = max(hi - lo, 0)
    if d <= k:
        return [int(x) for x in indices[lo:lo + d]]
    k0, k1 = split64(seed)
    taken = []
    for i in range(k):
        ctr = np.array([i, v, call & 0xFFFFFFFF, 0x70000000 | layer], np.uint32)
        u = int(philox4x32_10(ctr, np.array([k0, k1], np.uint32))[0])
        j = d - k + i
        t = (u * (j + 1)) >> 32
        taken.append(j if t in taken else t)
    return [int(indices[lo + p]) for p in sorted(taken)]


def rows_graph(degrees, N=None, seed=0):
    """A CSR with the given row lengths, entries drawn over [-2, N + 3) (out-of-range ones included) with duplicates and
    self loops."""
    r = np.random.RandomState(seed)
    N = len(degrees) if N is None else N
    indptr = np.concatenate([[0], np.cumsum(degrees)]).astype(np.int64)
    indices = r.randint(-2, N + 3, size=int(indptr[-1])).astype(np.int32)
    for v in range(min(N, len(degrees))):
        if degrees[v] > 3:
            indices[indptr[v]] = v                            # a self loop
            indices[indptr[v] + 1] = indices[indptr[v] + 2]  # a duplicate
    return indptr, indices


# ---------------------------------------------------------------- the sample
@pytest.mark.parametrize("k", [1, 3, 10, 25, 256])
def test_sample_rows_equal_the_scalar_restatement(k):
    degrees = [0, 1, k - 1 if k > 1 else 0, k, k + 1, 2 * k + 3, 600, 5, 0, 300]
    indptr, indices = rows_graph(degrees)
    for seed, call, layer in [(0, 0, 0), (123, 7, 1), (2**63 + 5, 2**40 + 3, 7)]:
        s_ptr, s_idx = sb.sample_rows(indptr, indices, k, seed, call, layer)
        assert s_ptr[0] == 0 and np.array_equal(np.diff(s_ptr), np.minimum(degrees, k))
        for v in range(len(degrees)):
            got = s_idx[s_ptr[v]:s_ptr[v + 1]].tolist()
            assert got == scalar_sample(indptr, indices, v, k, seed, call, layer), (k, v, seed)


def test_floyd_moves():
    # d = k + 1: step 0 draws t in [0, 1], step i in [0, i + 1]; every position distinct, all in range
    u = sb.draws(np.arange(500), 4, 9, 0, 0)
    held = sb.floyd_positions(u, np.full(500, 5))
    assert np.all(np.sort(held, 1)[:, 1:] != np.sort(held, 1)[:, :-1]) and held.min() >= 0 and held.max() <= 4
    # a taken t falls back to j: with u = 0 every step draws t = 0
    held = sb.floyd_positions(np.zeros((1, 4), np.uint32), np.array([10]))
    assert held.tolist() == [[0, 7, 8, 9]]
    # u = 2^32 - 1 draws t = j: never a collision
    held = sb.floyd_positions(np.full((1, 3), 2**32 - 1, np.uint32), np.array([9]))
    assert held.tolist() == [[6, 7, 8]]


def test_sample_words_and_nodes_subset():
    indptr, indices = rows_graph([40] * 6)
    full = sb.sample_rows(indptr, indices, 5, 1, 2, 3)
    part = sb.sample_rows(indptr, indices, 5, 1, 2, 3, nodes=[4, 1, 1, -1, 99])
    for v in range(6):
        a = full[1][full[0][v]:full[0][v + 1]]
        b = part[1][part[0][v]:part[0][v + 1]]
        assert np.array_equal(a, b) if v in (1, 4) else len(b) == 0
    # the layer, the call and the node each select other words
    for other in [(1, 2, 4), (1, 3, 3), (2, 2, 3)]:
        assert not np.array_equal(full[1], sb.sample_rows(indptr, indices, 5, *other)[1])


def test_fanout_range():
    indptr, indices = rows_graph([3, 4])
    for k in (0, -1, 257):
        with pytest.raises(ValueError, match="fanout"):
            sb.sample_rows(indptr, indices, k, 0, 0, 0)
        with pytest.raises(ValueError, match="fanout"):
            sb.sampled_blocks(indptr, indices, [0], [k], 0, 0)
        with pytest.raises(ValueError, match="fanout"):
            ops.check_fanouts([k], 1)
    with pytest.raises(ValueError, match="one entry per layer"):
        ops.check_fanouts([3, 4], 1)
    assert ops.check_fanouts([1, 256], 2) == [1, 256]


# ---------------------------------------------------------------- the blocks
@pytest.mark.parametrize("L", [1, 2, 3])
@pytest.mark.parametrize("fan", [1, 3, 256])
def test_block_invariants(L, fan):
    indptr, indices = hub_graph(N=60, seed=L)
    N = len(indptr) - 1
    fanouts = [fan, max(1, fan - 1), fan][:L]
    for seeds in (np.array([3, 3, -1, N, N + 5, 0, 17, 2]), np.arange(N), np.array([7]), np.zeros(0, np.int64)):
        blocks = sb.sampled_blocks(indptr, indices, seeds, fanouts, 11, 4)
        nxt = fb.clamp_ids(seeds, N)
        for l in range(L - 1, -1, -1):
            b = blocks[l]
            V = b["src_ids"].astype(np.int64)
            members = np.unique(nxt)
            assert np.all(np.diff(V) > 0) and V[-1] == N
            assert len(V) <= len(members) * (fanouts[l] + 1) + 1
            assert set(nxt.tolist()) <= set(V.tolist()) and np.array_equal(V[b["rows"]], nxt)
            s_ptr, s_idx = sb.sample_rows(indptr, indices, fanouts[l], 11, 4, l)
            for p, v in enumerate(V[:-1]):
                want = fb.clamp_ids(s_idx[s_ptr[v]:s_ptr[v + 1]], N) if v in set(members.tolist()) else []
                got = V[b["indices"][b["indptr"][p]:b["indptr"][p + 1]]]
                assert np.array_equal(got, want)
                assert len(got) == (min(max(indptr[v + 1] - indptr[v], 0), fanouts[l]) if v in members else 0)
            nxt = V


def test_large_fanouts_give_the_whole_neighbourhood_blocks():
    indptr, indices = hub_graph(N=60, seed=2)
    seeds = np.array([3, 3, -1, 60, 0, 17, 2])
    for L in (1, 2, 3):
        want = fb.csr_blocks(indptr, indices, seeds, L)
        got = sb.sampled_blocks(indptr, indices, seeds, [256] * L, 5, 9)
        for a, b in zip(got, want):
            for key in a:
                assert np.array_equal(a[key], b[key]) and a[key].dtype == b[key].dtype


def test_one_layer_is_the_whole_graph_over_the_sample():
    r = np.random.RandomState(3)
    indptr, indices = hub_graph(N=50, seed=4)
    N, F = len(indptr) - 1, 6
    x = r.randn(N + 1, F).astype(np.float32)
    x[N] = 0
    seeds = np.array([1, 4, 4, 7, 2, 49, -3])
    for kind in ("mean", "gcn", "maxpool"):
        aggs = _agg_dicts(kind, [F, 5], True, r)
        got = sb.sampled_embeddings(x, indptr, indices, aggs, True, seeds, [3], 8, 1)
        s_ptr, s_idx = sb.sample_rows(indptr, indices, 3, 8, 1, 0)
        want = fb.block_embeddings(x, s_ptr, s_idx, aggs, True, seeds)
        assert np.array_equal(got, want), kind


# float64 autograd of the whole-graph formula over S_0 (one layer: the block is the whole graph over the sample)
@pytest.mark.parametrize("kind,concat,d", [("mean", True, 0), ("gcn", False, 16), ("maxpool", True, 16),
                                           ("meanpool", False, 0)])
def test_gradients_equal_float64_autograd_over_the_sample(kind, concat, d):
    r = np.random.RandomState(9)
    indptr, indices = hub_graph(N=30, seed=3)
    N, F, C = len(indptr) - 1, 5, 3
    x = r.randn(N + 1, F).astype(np.float32)
    x[N] = 0
    feats = np.concatenate([r.randn(N + 1, d).astype(np.float32), x], 1) if d else x
    aggs = _agg_dicts(kind, [d + F, 4], concat, r)
    node_ids = np.array([0, 3, 5, 5, 9, 2, 11, 29], np.int64)
    out_w = 4 * (2 if concat and kind != "gcn" else 1)
    pred_w, pred_b = (r.randn(out_w, C) * 0.5).astype(np.float32), (r.randn(C) * 0.1).astype(np.float32)
    labels = np.eye(C)[r.randint(0, C, len(node_ids))]
    loss, grads, head, demb = sb.sampled_loss_grads(feats, indptr, indices, aggs, concat, node_ids, labels, pred_w,
                                                    pred_b, [2], 4, 0, False, 0.01, d)
    s_ptr, s_idx = sb.sample_rows(indptr, indices, 2, 4, 0, 0)
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


# ---------------------------------------------------------------- the law
def test_every_subset_equally_likely():
    n, d, k = 200000, 6, 3
    held = np.sort(sb.floyd_positions(sb.draws(np.arange(n), k, 77, 5, 2), np.full(n, d)), axis=1)
    code = (1 << held).sum(axis=1)
    counts = np.bincount(code, minlength=64)
    subsets = [c for c in range(64) if bin(c).count("1") == k]
    assert len(subsets) == 20 and counts[subsets].sum() == n
    p = 1.0 / 20
    sigma = np.sqrt(n * p * (1 - p))
    assert np.abs(counts[subsets] - n * p).max() < 5 * sigma, counts[subsets]


def test_inclusion_probability_on_a_hub_row():
    n, d, k = 4000, 1000, 25
    held = sb.floyd_positions(sb.draws(np.arange(n), k, 3, 0, 0), np.full(n, d))
    assert np.all(np.sort(held, 1)[:, 1:] > np.sort(held, 1)[:, :-1])
    counts = np.bincount(held.reshape(-1), minlength=d)
    p = k / d
    sigma = np.sqrt(n * p * (1 - p))
    assert np.abs(counts - n * p).max() < 5 * sigma
    chi2 = (((counts - n * p) ** 2) / (n * p)).sum()        # ~ d - 1 degrees of freedom
    assert abs(chi2 - (d - 1)) < 5 * np.sqrt(2 * (d - 1))


# ---------------------------------------------------------------- the autograd wiring, kernels replaced by the oracle
def _fake_sampled_blocks(indptr, indices, seeds, n_layers, fanouts=None, seed=0, call=0):
    if fanouts is None:
        return _fake_csr_blocks(indptr, indices, seeds, n_layers)
    assert len(fanouts) == n_layers
    return [ops.CsrBlock(*(torch.from_numpy(np.asarray(b[key])) for key in ("src_ids", "indptr", "indices", "rows")))
            for b in sb.sampled_blocks(_np(indptr), _np(indices), _np(seeds), fanouts, seed, call)]


@pytest.fixture()
def sampled_kernels(block_kernels, monkeypatch):
    monkeypatch.setattr(ops, "csr_blocks", _fake_sampled_blocks)


def _with_sampler(model, seed=5, counter=3):
    sampler = types.SimpleNamespace(seed=seed, counter=counter)
    for info in model.layer_infos:
        model.layer_infos[model.layer_infos.index(info)] = info._replace(neigh_sampler=sampler)
    return sampler


@pytest.mark.parametrize("kind,concat,d", [("mean", True, 0), ("gcn", False, 16), ("maxpool", True, 16),
                                           ("meanpool", False, 0)])
def test_supervised_wiring_matches_the_sampled_oracle(sampled_kernels, kind, concat, d):
    model, indptr, indices = _cpu_model(SupervisedGraphsage, kind, concat, d)
    sampler = _with_sampler(model)
    r = np.random.RandomState(2)
    node_ids = np.array([1, 4, 4, 7, 2, 39, -3], np.int64)
    labels = np.eye(3)[r.randint(0, 3, len(node_ids))]
    loss = model.sampled_minibatch_loss(indptr, indices, node_ids, labels)
    assert sampler.counter == 4
    loss.backward()
    fanouts = [info.num_samples for info in model.layer_infos]
    rl, grads, head, demb = sb.sampled_loss_grads(_np(model.features), indptr, indices, fnt_oracle_dicts(model), concat,
                                                  fb.clamp_ids(node_ids, len(indptr) - 1), labels,
                                                  _np(model.node_pred_vars["weights"]), _np(model.node_pred_vars["bias"]),
                                                  fanouts, 5, 3, False, 0.01, d)
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
        emb = model.sampled_minibatch_embeddings(indptr, indices, node_ids)          # call 4
    want = sb.sampled_embeddings(_np(model.features), indptr, indices, fnt_oracle_dicts(model), concat, node_ids,
                                 fanouts, 5, 4)
    assert np.abs(_np(emb) - want).max() < 1e-5 and sampler.counter == 5
    before = [p.detach().clone() for p in model.parameters()]
    model.sampled_minibatch_train_step(indptr, indices, node_ids, labels)
    assert sampler.counter == 6
    assert any(not torch.equal(a, p.detach()) for a, p in zip(before, model.parameters()))


def fnt_oracle_dicts(model):
    from test_full_neighbor_train_cpu import oracle_dicts
    return oracle_dicts(model)


def test_unsupervised_wiring(sampled_kernels):
    model, indptr, indices = _cpu_model(UnsupervisedGraphsage, "mean", True, 0, neg_sample_size=4)
    sampler = _with_sampler(model, seed=9, counter=0)
    model.neg_sampler = _FakeNegatives([5, 0, 33, 5])
    b1, b2 = np.array([1, 2, 3, 9]), np.array([4, 4, 38, 0])
    loss = model.sampled_minibatch_loss(indptr, indices, b1, b2)
    assert model.neg_sampler.counter == 1 and sampler.counter == 1
    loss.backward()
    assert np.isfinite(float(model.mrr()))
    # the same loss from one set of sampled blocks over cat(b1, b2, neg) at call 0
    sampler.counter = 0
    model.optimizer.zero_grad(set_to_none=True)
    out = fnt.full_neighbor_outputs(model, indptr, indices, torch.cat([torch.tensor(b1), torch.tensor(b2),
                                                                       model.neg_sampler.ids.long()]),
                                    minibatch=True, sampled=True)
    want = model._pairs_loss(*torch.split(out, [4, 4, 4]))
    assert torch.equal(loss.detach(), want.detach())
    model.sampled_minibatch_train_step(indptr, indices, b1, b2)
    assert model.neg_sampler.counter == 2 and sampler.counter == 2


# ---------------------------------------------------------------- refusals (no GPU needed: they fire first)
def _sampled_bare(kind="mean", **attrs):
    m = _bare_model(kind, **attrs)
    m.layer_infos = [types.SimpleNamespace(num_samples=3, neigh_sampler=types.SimpleNamespace(seed=1, counter=0))]
    return m


def test_refusals(monkeypatch):
    with pytest.raises(NotImplementedError, match="seq"):
        _sampled_bare("seq").sampled_minibatch_train_step(*CSR, [0], [[1.0]])
    with pytest.raises(NotImplementedError, match="seq"):
        _sampled_bare("seq").sampled_minibatch_embeddings(*CSR, [0])
    m = _sampled_bare()
    m.features = type("Sharded", (), {"c_table": lambda self: None, "shape": (5, 3)})()
    with pytest.raises(NotImplementedError, match="ShardedFeatures"):
        m.sampled_minibatch_loss(*CSR, [0], [[1.0]])
    with pytest.raises(NotImplementedError, match="distributed"):
        _sampled_bare(distributed=True).sampled_minibatch_outputs(*CSR, [0])
    m = _sampled_bare(dropout_rate=0.5)
    with pytest.raises(NotImplementedError, match="dropout"):
        m.sampled_minibatch_train_step(*CSR, [0], [[1.0]])
    assert m.layer_infos[0].neigh_sampler.counter == 0                   # refused before any draw
    u = UnsupervisedGraphsage.__new__(UnsupervisedGraphsage)
    u.__dict__.update(_sampled_bare(dropout_rate=0.1).__dict__)
    u.neg_sampler = _FakeNegatives([0])
    with pytest.raises(NotImplementedError, match="dropout"):
        u.sampled_minibatch_train_step(*CSR, [0], [1])
    assert u.neg_sampler.counter == 0                                     # refused before drawing negatives
    m = _sampled_bare()
    m.layer_infos[0].num_samples = 300
    m.aggregators = []
    with pytest.raises(ValueError, match="fanout"):
        m.sampled_minibatch_embeddings(*CSR, [0])
    assert m.layer_infos[0].neigh_sampler.counter == 0
    monkeypatch.setattr(torch.cuda, "is_available", lambda: True)
    monkeypatch.setattr(torch.cuda, "is_current_stream_capturing", lambda: True)
    with pytest.raises(NotImplementedError, match="CUDA graph"):
        _sampled_bare().sampled_minibatch_train_step(*CSR, [0], [[1.0]])
    with pytest.raises(NotImplementedError, match="CUDA graph"):
        _sampled_bare(aggregators=[]).sampled_minibatch_embeddings(*CSR, [0])


def test_kernels_have_no_cpu_fallback():
    with pytest.raises(RuntimeError, match="CUDA-only"):
        ops.csr_blocks(torch.zeros(3, dtype=torch.int64), torch.zeros(0, dtype=torch.int32),
                       torch.zeros(1, dtype=torch.int32), 2, fanouts=[3, 3])
    with pytest.raises(RuntimeError, match="CUDA-only"):
        ops.sample_csr_rows(torch.zeros(3, dtype=torch.int64), torch.zeros(0, dtype=torch.int32), 3, 0, 0, 0)
