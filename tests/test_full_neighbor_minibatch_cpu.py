"""Minibatches over whole neighbourhoods without a GPU: the block contract (oracle/full_neighbor_blocks.py) against the
whole-graph oracle bit for bit, the blocks' invariants, the gradients through the blocks against float64 torch autograd of
the whole-graph formula, the autograd wiring of full_neighbor_minibatch_* for both models with the oracle standing in for
the kernels (TEST mocks only: the product has no such path), and the refusals."""
import numpy as np
import pytest
import torch

import graphsage_b200 as gs
from graphsage_b200 import full_neighbor_training as fnt
from graphsage_b200 import ops
from graphsage_b200.supervised_models import SupervisedGraphsage
from graphsage_b200.unsupervised_models import UnsupervisedGraphsage
from oracle import full_neighbor as fn
from oracle import full_neighbor_blocks as fb
from oracle import numerics as nu
from test_full_neighbor_train_cpu import (CSR, _agg_dicts, _bare_model, _np, _torch_formula, cpu_kernels,  # noqa: F401
                                          messy_graph, oracle_dicts)


def hub_graph(N=60, seed=0):
    """messy_graph's rows (empty rows, duplicates, self loops, out-of-range entries, a long row) plus an in-degree hub:
    node 4 in half of the rows."""
    indptr, indices = messy_graph(N, seed)
    rows = [list(indices[indptr[i]:indptr[i + 1]]) + ([4] if i % 2 else []) for i in range(N)]
    indptr = np.concatenate([[0], np.cumsum([len(r) for r in rows])]).astype(np.int64)
    return indptr, np.array([x for r in rows for x in r], dtype=np.int32)


def seed_cases(N):
    return {"mixed": np.array([3, 3, -1, N, N + 5, 0, 17, 2], np.int64),   # duplicates, out of range, the dummy, the long row
            "every node": np.arange(N), "single": np.array([7]), "empty row": np.array([3]),
            "none": np.zeros(0, np.int64)}


# ---------------------------------------------------------------- the blocks
@pytest.mark.parametrize("L", [1, 2, 3])
@pytest.mark.parametrize("case", ["mixed", "every node", "single", "empty row", "none"])
def test_block_invariants(L, case):
    indptr, indices = hub_graph()
    N = len(indptr) - 1
    seeds = seed_cases(N)[case]
    blocks = fb.csr_blocks(indptr, indices, seeds, L)
    assert len(blocks) == L
    nxt = fb.clamp_ids(seeds, N)
    for l in range(L - 1, -1, -1):
        b = blocks[l]
        V = b["src_ids"].astype(np.int64)
        assert np.all(np.diff(V) > 0) and V[-1] == N                             # ascending, unique, the dummy last
        assert set(nxt.tolist()) <= set(V.tolist())                              # V_{l+1} is in V_l
        assert np.array_equal(V[b["rows"]], nxt)                                 # rows name the next level's nodes
        assert len(b["indptr"]) == len(V) and b["indptr"][0] == 0 and np.all(np.diff(b["indptr"]) >= 0)
        members = set(nxt.tolist())
        for p, v in enumerate(V[:-1]):                                           # raw rows of members, relabelled
            want = fb.clamp_ids(indices[indptr[v]:indptr[v + 1]], N) if v in members else np.zeros(0, np.int64)
            assert np.array_equal(V[b["indices"][b["indptr"][p]:b["indptr"][p + 1]]], want)
        assert b["indptr"][-1] == len(b["indices"])
        nxt = V


@pytest.mark.parametrize("L", [1, 2, 3])
@pytest.mark.parametrize("concat", [False, True])
@pytest.mark.parametrize("kind", ["mean", "gcn", "maxpool", "meanpool"])
def test_block_embeddings_equal_the_whole_graph_bit_for_bit(kind, concat, L):
    r = np.random.RandomState(L + 7 * concat)
    indptr, indices = hub_graph(seed=L)
    N, F = len(indptr) - 1, 7
    x = r.randn(N + 1, F).astype(np.float32)
    x[N] = 0
    aggs = _agg_dicts(kind, [F] + [6] * L, concat, r)
    for case, seeds in seed_cases(N).items():
        got = fb.block_embeddings(x, indptr, indices, aggs, concat, seeds)
        want = fn.full_neighbor_embeddings(x, indptr, indices, aggs, concat, node_ids=fb.clamp_ids(seeds, N))
        assert got.shape == want.shape and nu.bits_equal(got, want), (case, kind, concat, L)


# float64 autograd of the whole-graph formula, on the seeds' loss
GRAD_CASES = [("mean", True, 0, 2, False, False), ("gcn", False, 16, 2, False, True), ("maxpool", True, 0, 2, True, False),
              ("maxpool", False, 16, 2, False, True), ("meanpool", True, 16, 2, False, False),
              ("mean", False, 16, 1, False, False), ("gcn", True, 0, 3, False, False), ("maxpool", True, 16, 3, True, True)]


@pytest.mark.parametrize("kind,concat,d,L,integer,sigmoid", GRAD_CASES)
def test_block_gradients_equal_float64_autograd(kind, concat, d, L, integer, sigmoid):
    r = np.random.RandomState(9)
    indptr, indices = hub_graph(N=30, seed=3)
    N, F, C = len(indptr) - 1, 5, 3
    x = r.randint(0, 3, size=(N + 1, F)).astype(np.float32) if integer else r.randn(N + 1, F).astype(np.float32)
    x[N] = 0
    feats = np.concatenate([r.randn(N + 1, d).astype(np.float32), x], 1) if d else x
    aggs = _agg_dicts(kind, [d + F] + [4] * L, concat, r, integer)
    node_ids = np.array([0, 3, 5, 5, 9, 2, 11, 29], np.int64)
    out_w = 4 * (2 if concat and kind != "gcn" else 1)
    pred_w, pred_b = (r.randn(out_w, C) * 0.5).astype(np.float32), (r.randn(C) * 0.1).astype(np.float32)
    labels = (r.rand(len(node_ids), C) > 0.5).astype(np.float64) if sigmoid else np.eye(C)[r.randint(0, C, len(node_ids))]
    loss, grads, head, demb = fb.block_loss_grads(feats, indptr, indices, aggs, concat, node_ids, labels, pred_w, pred_b,
                                                  sigmoid, 0.01, d)
    rl, rgrads, rhead, rdemb = _torch_formula(feats, indptr, indices, aggs, concat, node_ids, pred_w, pred_b, labels,
                                              sigmoid, 0.01, d)
    assert abs(loss - rl) < 1e-5 * max(1, abs(rl))

    def close(a, b, what):
        assert a.shape == b.shape, what
        assert np.abs(a - b).max() <= 1e-4 * max(1.0, np.abs(b).max()), (what, np.abs(a - b).max())
    for l, (g, rg) in enumerate(zip(grads, rgrads)):
        assert set(g) == set(rg)
        for k in g:
            close(g[k], rg[k], (l, k))
    close(head["weights"], rhead["weights"], "head")
    if d:
        close(demb, rdemb, "embeddings")


# ---------------------------------------------------------------- the autograd wiring, kernels replaced by the oracle
class _FakeTableRows(object):
    def __init__(self, table, ranges, M):
        (ids, row0), = ranges
        self.rows = table[torch.where((ids < 0) | (ids >= table.shape[0]), table.shape[0] - 1, ids).long()]


def _fake_sage_gemm(parts, combine=ops.COMBINE_ADD, bias=None, act=ops.ACT_NONE, math=None, out=None, packed=None):
    ys = [(a.rows if isinstance(a, _FakeTableRows) else a)[:, :k] @ w for (a, k, w) in parts]
    y = torch.cat(ys, dim=1) if combine == ops.COMBINE_CONCAT else sum(ys[1:], ys[0])
    if bias is not None:
        y = y + bias
    return torch.relu(y) if act == ops.ACT_RELU else y


def _fake_csr_blocks(indptr, indices, seeds, n_layers):
    return [ops.CsrBlock(*(torch.from_numpy(b[k]) for k in ("src_ids", "indptr", "indices", "rows")))
            for b in fb.csr_blocks(_np(indptr), _np(indices), _np(seeds), n_layers)]


@pytest.fixture()
def block_kernels(cpu_kernels, monkeypatch):
    monkeypatch.setattr(ops, "sage_gemm", _fake_sage_gemm)
    monkeypatch.setattr(ops, "TableRows", _FakeTableRows)
    monkeypatch.setattr(ops, "csr_blocks", _fake_csr_blocks)
    monkeypatch.setattr(ops, "gather_rows_f32", lambda feats, ids=None, row0=0, n=None, out=None:
                        feats[ids.long()].float().clone())


def _cpu_model(cls, kind, concat, d, C=3, **kw):
    r = np.random.RandomState(11)
    indptr, indices = hub_graph(N=40, seed=5)
    N, F = len(indptr) - 1, 6
    feats = np.vstack([r.randn(N, F).astype(np.float32), np.zeros((1, F), np.float32)])
    infos = [gs.SAGEInfo("node", None, 3, 8), gs.SAGEInfo("node", None, 3, 8)]
    adj = torch.zeros((N + 1, 3), dtype=torch.int32)
    args = (C, {}) if cls is SupervisedGraphsage else ({},)
    model = cls(*args, torch.from_numpy(feats), adj, None if cls is SupervisedGraphsage else np.ones(N + 1), infos,
                concat=concat, aggregator_type=kind, identity_dim=d, weight_decay=0.01, device="cpu", **kw)
    model.aggregator_type = kind
    for a in model.aggregators:
        a.math = ops.MATH_FP32_SIMT
    return model, indptr, indices


def _grads(model):
    return [None if p.grad is None else p.grad.clone() for p in model.parameters()]


@pytest.mark.parametrize("kind,concat,d", [("mean", True, 0), ("gcn", False, 16), ("maxpool", True, 16),
                                           ("meanpool", False, 0)])
def test_supervised_wiring_matches_the_block_oracle(block_kernels, kind, concat, d):
    model, indptr, indices = _cpu_model(SupervisedGraphsage, kind, concat, d)
    r = np.random.RandomState(2)
    node_ids = np.array([1, 4, 4, 7, 2, 39, -3], np.int64)
    labels = np.eye(3)[r.randint(0, 3, len(node_ids))]
    out = model.full_neighbor_minibatch_outputs(indptr, indices, node_ids)
    assert torch.equal(out.detach(), model.full_neighbor_outputs(indptr, indices, node_ids).detach())
    loss = model.full_neighbor_minibatch_loss(indptr, indices, node_ids, labels)
    loss.backward()
    rl, grads, head, demb = fb.block_loss_grads(_np(model.features), indptr, indices, oracle_dicts(model), concat,
                                                fb.clamp_ids(node_ids, len(indptr) - 1), labels,
                                                _np(model.node_pred_vars["weights"]), _np(model.node_pred_vars["bias"]),
                                                False, 0.01, d)
    assert abs(float(loss.detach()) - rl) < 1e-5

    def close(t, ref, what):
        assert t.grad is not None, what
        assert np.abs(_np(t.grad) - ref).max() <= 1e-4 * max(1.0, np.abs(ref).max()), what
    for a, g in zip(model.aggregators, grads):
        for k, v in a.vars.items():
            close(v, g[k], k)
        if hasattr(a, "mlp_layers"):
            close(a.mlp_layers[0].vars["weights"], g["mlp_weights"], "mlp_weights")
            close(a.mlp_layers[0].vars["bias"], g["mlp_bias"], "mlp_bias")
    close(model.node_pred_vars["weights"], head["weights"], "head")
    if d:
        close(model.embeds, demb, "embeds")
    before = [p.detach().clone() for p in model.parameters()]
    model.full_neighbor_minibatch_train_step(indptr, indices, node_ids, labels)
    assert any(not torch.equal(a, p.detach()) for a, p in zip(before, model.parameters()))


class _FakeNegatives(object):
    def __init__(self, ids):
        self.ids, self.counter = torch.tensor(ids, dtype=torch.int32), 0

    def __call__(self, num_sampled):
        self.counter += 1
        return self.ids[:num_sampled]


@pytest.mark.parametrize("kind,d", [("mean", 16), ("maxpool", 0), ("gcn", 0)])
def test_unsupervised_wiring_matches_the_whole_graph_loss(block_kernels, kind, d):
    model, indptr, indices = _cpu_model(UnsupervisedGraphsage, kind, kind != "gcn", d, neg_sample_size=4)
    model.neg_sampler = _FakeNegatives([5, 0, 33, 5])
    b1, b2 = np.array([1, 2, 3, 9]), np.array([4, 4, 38, 0])
    loss = model.full_neighbor_minibatch_loss(indptr, indices, b1, b2)
    assert model.neg_sampler.counter == 1
    loss.backward()
    got = _grads(model)
    mrr = float(model.mrr())
    # the same loss from the whole-graph outputs with the same negatives
    model.optimizer.zero_grad(set_to_none=True)
    out = fnt.full_neighbor_outputs(model, indptr, indices, torch.cat([torch.tensor(b1), torch.tensor(b2),
                                                                       model.neg_sampler.ids.long()]))
    o1, o2, on = torch.split(out, [4, 4, 4])
    want = model.link_pred_layer.loss(o1, o2, on) + gs.supervised_models.weight_decay_term(model.decayed_parameters(),
                                                                                            0.01)
    (want / 4.0).backward()
    assert torch.equal(loss.detach(), (want / 4.0).detach())
    for a, p in zip(got, model.parameters()):
        assert (a is None) == (p.grad is None)
        if a is not None:
            assert torch.allclose(a, p.grad, rtol=1e-4, atol=1e-6)
    assert np.isfinite(mrr)
    model.full_neighbor_minibatch_train_step(indptr, indices, b1, b2)
    assert model.neg_sampler.counter == 2


# ---------------------------------------------------------------- refusals (no GPU needed: they fire first)
def test_refusals(monkeypatch):
    with pytest.raises(NotImplementedError, match="seq"):
        _bare_model("seq").full_neighbor_minibatch_train_step(*CSR, [0], [[1.0]])
    with pytest.raises(NotImplementedError, match="seq"):
        _bare_model("seq").full_neighbor_minibatch_embeddings(*CSR, [0])
    m = _bare_model()
    m.features = type("Sharded", (), {"c_table": lambda self: None, "shape": (5, 3)})()
    with pytest.raises(NotImplementedError, match="ShardedFeatures"):
        m.full_neighbor_minibatch_loss(*CSR, [0], [[1.0]])
    with pytest.raises(NotImplementedError, match="ShardedFeatures"):
        m.full_neighbor_minibatch_embeddings(*CSR, [0])
    with pytest.raises(NotImplementedError, match="distributed"):
        _bare_model(distributed=True).full_neighbor_minibatch_outputs(*CSR, [0])
    with pytest.raises(NotImplementedError, match="dropout"):
        _bare_model(dropout_rate=0.5).full_neighbor_minibatch_train_step(*CSR, [0], [[1.0]])
    with pytest.raises(ValueError, match="N \\+ 1"):
        _bare_model().full_neighbor_minibatch_loss(np.zeros(4, np.int64), np.zeros(0, np.int32), [0], [[1.0]])
    u = UnsupervisedGraphsage.__new__(UnsupervisedGraphsage)
    u.__dict__.update(_bare_model().__dict__)
    u.neg_sampler = _FakeNegatives([0])
    u.distributed = True
    with pytest.raises(NotImplementedError, match="distributed"):
        u.full_neighbor_minibatch_train_step(*CSR, [0], [1])
    assert u.neg_sampler.counter == 0                                     # refused before drawing negatives
    monkeypatch.setattr(torch.cuda, "is_available", lambda: True)
    monkeypatch.setattr(torch.cuda, "is_current_stream_capturing", lambda: True)
    with pytest.raises(NotImplementedError, match="CUDA graph"):
        _bare_model().full_neighbor_minibatch_train_step(*CSR, [0], [[1.0]])
    with pytest.raises(NotImplementedError, match="CUDA graph"):
        _bare_model(aggregators=[]).full_neighbor_minibatch_embeddings(*CSR, [0])


def test_csr_blocks_has_no_cpu_fallback_and_checks_its_inputs():
    with pytest.raises(RuntimeError, match="CUDA-only"):
        ops.csr_blocks(torch.zeros(3, dtype=torch.int64), torch.zeros(0, dtype=torch.int32),
                       torch.zeros(1, dtype=torch.int32), 2)
