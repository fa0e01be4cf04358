"""Node2Vec / DeepWalk baseline (reference graphsage/models.py:408-501) on the CPU: the oracle against the fixture written
by the reference's own Node2VecModel (tests/golden/make_n2v_golden.py), the oracle's gradients and SGD step against torch
autograd, the unique unigram sampler's contract, and the host side of the two-phase (train, then retrain on val/test walk
pairs) flow on the toy-ppi slice."""
import os
import random

import numpy as np
import pytest
import torch

from graphsage_b200 import minibatch, utils
from graphsage_b200.graph import Graph
from graphsage_b200.node2vec import Node2VecModel, check_unique_sample_size
from graphsage_b200.prediction import mrr_from_affinities
from oracle import node2vec as on2v

HERE = os.path.dirname(os.path.abspath(__file__))


def cases(golden):
    g = golden("n2v")
    for ci in range(int(g["n_cases"])):
        yield {k[len("c%d_" % ci):]: g[k] for k in g.files if k.startswith("c%d_" % ci)}


# ------------------------------------------------------------------ the oracle against the reference's own code
def test_oracle_matches_reference_node2vec(golden):
    for c in cases(golden):
        B, S = len(c["batch1"]), len(c["neg"])
        neg = on2v.sample_unigram_unique(c["deg"], S, int(c["seed"]), int(c["counter"]))
        assert np.array_equal(neg, c["neg"])
        loss, aff, neg_aff = on2v.skipgram_forward(c["T"], c["C"], c["b"], c["batch1"], c["batch2"], c["neg"])
        assert abs(loss - float(c["loss"])) <= 1e-5 * abs(float(c["loss"]))            # bias in the loss, / the short B
        # the MRR table is [neg..., true] WITHOUT the biases
        assert np.allclose(c["aff_all"][:, :S], neg_aff, rtol=1e-5, atol=1e-5)
        assert np.allclose(c["aff_all"][:, S], aff, rtol=1e-5, atol=1e-5)
        rank, mrr = on2v.ranks(c["aff_all"][:, S], c["aff_all"][:, :S])
        assert np.array_equal(rank, c["ranks"])
        assert abs(mrr - float(c["mrr"])) < 1e-6
        assert abs(float(mrr_from_affinities(torch.from_numpy(c["aff_all"][:, S]), torch.from_numpy(c["aff_all"][:, :S])))
                   - float(c["mrr"])) < 1e-6
        assert np.array_equal(c["outputs1"], c["T"][c["batch1"]])
        # what the fixture pins is not satisfied by the wrong variants
        wrong_b = on2v.skipgram_forward(c["T"], c["C"], np.zeros_like(c["b"]), c["batch1"], c["batch2"], c["neg"])[0]
        assert abs(wrong_b - float(c["loss"])) > 1e-3
        assert abs(loss * B / 512 - float(c["loss"])) > 1e-3


def test_fixture_has_the_duplicates_it_should(golden):
    for c in cases(golden):
        assert len(set(c["batch1"].tolist())) < len(c["batch1"])
        assert len(set(c["batch2"].tolist())) < len(c["batch2"])
        assert set(c["batch2"].tolist()) & set(c["neg"].tolist())
        assert len(c["batch1"]) < 512                                                # a short batch


# ------------------------------------------------------------------ gradients and the SGD step against torch autograd
def _torch_loss(T, C, b, batch1, batch2, neg):
    t, c, n = T[batch1], C[batch2], C[neg]
    aff = (t * c).sum(1) + b[batch2]
    neg_aff = t @ n.t() + b[neg][None, :]
    return (torch.nn.functional.softplus(-aff).sum() + torch.nn.functional.softplus(neg_aff).sum()) / len(batch1)


def test_oracle_gradients_and_sgd_step_vs_torch_autograd(golden):
    lr = 0.37
    for c in cases(golden):
        b1, b2, neg = (torch.from_numpy(c[k].astype(np.int64)) for k in ("batch1", "batch2", "neg"))
        T, C, b = (torch.from_numpy(c[k].astype(np.float64)) for k in ("T", "C", "b"))
        # per-lookup gradients: differentiate w.r.t. the looked-up rows
        t, cc, n = T[b1].requires_grad_(), C[b2].requires_grad_(), C[neg].requires_grad_()
        cb, nb = b[b2].requires_grad_(), b[neg].requires_grad_()
        aff = (t * cc).sum(1) + cb
        neg_aff = t @ n.t() + nb[None, :]
        loss = (torch.nn.functional.softplus(-aff).sum() + torch.nn.functional.softplus(neg_aff).sum()) / len(b1)
        loss.backward()
        g = on2v.skipgram_grads(c["T"], c["C"], c["b"], c["batch1"], c["batch2"], c["neg"])
        for mine, ref in ((g["gt"], t.grad), (g["gc_pos"], cc.grad), (g["gb_pos"], cb.grad), (g["gc_neg"], n.grad),
                          (g["gb_neg"], nb.grad)):
            assert np.allclose(mine, ref.numpy(), rtol=1e-12, atol=1e-14)
        # the update: dense autograd gradients of the tables (duplicates summed) == index_add_ of the lookup gradients
        Tl, Cl, bl = T.clone().requires_grad_(), C.clone().requires_grad_(), b.clone().requires_grad_()
        _torch_loss(Tl, Cl, bl, b1, b2, neg).backward()
        T2 = T.clone().index_add_(0, b1, torch.from_numpy(g["gt"]), alpha=-lr)
        C2 = C.clone().index_add_(0, b2, torch.from_numpy(g["gc_pos"]), alpha=-lr).index_add_(0, neg, torch.from_numpy(g["gc_neg"]),
                                                                                          alpha=-lr)
        bb2 = b.clone().index_add_(0, b2, torch.from_numpy(g["gb_pos"]), alpha=-lr).index_add_(0, neg, torch.from_numpy(g["gb_neg"]),
                                                                                           alpha=-lr)
        assert torch.allclose(T2, T - lr * Tl.grad) and torch.allclose(C2, C - lr * Cl.grad) and torch.allclose(bb2, b - lr * bl.grad)
        To, Co, bo, loss0 = on2v.sgd_step(c["T"], c["C"], c["b"], c["batch1"], c["batch2"], c["neg"], lr)
        assert np.allclose(To, T2.numpy(), rtol=0, atol=1e-12) and np.allclose(Co, C2.numpy(), rtol=0, atol=1e-12)
        assert np.allclose(bo, bb2.numpy(), rtol=0, atol=1e-12)
        assert abs(loss0 - float(loss.detach())) < 1e-12
        untouched = np.setdiff1d(np.arange(len(c["T"])), np.concatenate([c["batch1"]]))
        assert np.array_equal(To[untouched], c["T"][untouched].astype(np.float64))


# ------------------------------------------------------------------ the unique unigram sampler
def _hub_degrees(n=50, hub=1e6):
    deg = np.ones(n)
    deg[7] = hub
    deg[3] = 0.0
    return deg


@pytest.mark.parametrize("deg, S", [(np.arange(1, 300, dtype=np.float64), 20), (np.arange(1, 300, dtype=np.float64), 299),
                                    (_hub_degrees(), 20), (_hub_degrees(), 49), (np.r_[np.zeros(5), np.ones(3)], 3)])
def test_unique_sampler_contract(deg, S):
    for seed, counter in ((123, 0), (123, 1), (9, 1 << 40)):
        out = on2v.sample_unigram_unique(deg, S, seed, counter)
        assert len(out) == S and len(set(out.tolist())) == S and (out >= 0).all()
        assert (deg[out] > 0).all()
        # the kernel's 32-lane rounds give the literal loop's result
        assert np.array_equal(on2v.sample_unigram_unique_rounds(deg, S, seed, counter), out)
        # first-occurrence order of the raw draw sequence
        raw = on2v.raw_unigram_draws(on2v.unigram_cdf(deg), seed, counter, 0, 1 << 16)
        _, first = np.unique(raw, return_index=True)
        k = min(S, len(first))                          # (the hub case needs more than 2^16 draws for all of them)
        assert k >= min(S, 20) and np.array_equal(raw[np.sort(first)][:k], out[:k])
        assert np.array_equal(on2v.sample_unigram_unique(deg, S, seed, counter), out)        # determinism
    assert not np.array_equal(on2v.sample_unigram_unique(deg, S, 123, 0), on2v.sample_unigram_unique(deg, S, 123, 1)) or S == 3


def test_unique_sampler_refuses_more_than_the_support():
    deg = np.r_[np.zeros(5), np.ones(3)]
    with pytest.raises(ValueError):
        on2v.sample_unigram_unique(deg, 4, 1, 0)
    with pytest.raises(ValueError):
        check_unique_sample_size(deg, 4)
    check_unique_sample_size(deg, 3)
    with pytest.raises(ValueError):
        check_unique_sample_size(np.ones(5000), 1025)
    # the model refuses before touching a device
    with pytest.raises(ValueError):
        Node2VecModel({}, 8, deg, nodevec_dim=4, neg_sample_size=4, device="cpu")
    with pytest.raises(ValueError):
        Node2VecModel({}, 7, np.ones(8), nodevec_dim=4, neg_sample_size=4, device="cpu")


def test_budget_exhaustion_is_reported_not_looped():
    deg = np.r_[1e15, 1.0]                                # the second id is (almost) never drawn
    out = on2v.sample_unigram_unique(deg, 2, 5, 0, budget=4096)
    assert out[0] == 0 and out[1] == -1


# ------------------------------------------------------------------ the two-phase flow's host logic on toy-ppi
def toy_graph(bridges=60):
    """The toy-ppi slice as a Graph (node kinds, links with train_removed) and its id map.  The slice was cut breadth-first
    inside each node kind, so it has no val/test - train links; `bridges` of them (train_removed, as every link that
    touches a val/test node is in the dataset) are added, every 5th val/test node to a train node, so that walks started
    at val/test nodes reach the train graph as they do on the whole dataset."""
    d = np.load(os.path.join(HERE, "golden", "toy_ppi.npz"))
    G = Graph()
    ids = [int(u) for u in d["ids"]]
    for u, v, t in zip(ids, d["val"], d["test"]):
        G.add_node(u, val=bool(v), test=bool(t))
    for a, b, rm in zip(d["src"], d["dst"], d["train_removed"]):
        G.add_edge(ids[int(a)], ids[int(b)])
        G[ids[int(a)]][ids[int(b)]]["train_removed"] = bool(rm)
    train = [u for u, v, t in zip(ids, d["val"], d["test"]) if not v and not t]
    other = [u for u, v, t in zip(ids, d["val"], d["test"]) if v or t]
    for k in range(bridges):
        u, v = other[5 * k % len(other)], train[7 * k % len(train)]
        G.add_edge(u, v)
        G[u][v]["train_removed"] = True
    return G, {u: i for i, u in enumerate(sorted(ids))}


def two_phase_iterators(G, id_map, batch_size=512, walks=2, seed=5):
    """Phase 1: walk pairs over the train graph (what -walks.txt holds, utils.py:95-106); phase 2: walk pairs started
    at the val/test nodes over the whole graph, retrained with n2v_retrain / fixed_n2v (unsupervised_train.py:337-354)."""
    train = [n for n in G.nodes() if not G.node[n]["val"] and not G.node[n]["test"]]
    rng = random.Random(seed)
    pairs1 = utils.run_random_walks(G.subgraph(train), train, num_walks=walks, rng=rng)
    np.random.seed(seed)
    it1 = minibatch.EdgeMinibatchIterator(G, id_map, None, context_pairs=pairs1, batch_size=batch_size, max_degree=25)
    test_nodes = [n for n in G.nodes() if G.node[n]["val"] or G.node[n]["test"]]
    pairs2 = utils.run_random_walks(G, test_nodes, num_walks=walks, rng=rng)
    it2 = minibatch.EdgeMinibatchIterator(G, id_map, None, context_pairs=pairs2, batch_size=batch_size, max_degree=25,
                                          n2v_retrain=True, fixed_n2v=True)
    return it1, it2


def test_two_phase_flow_host_logic_on_toy_ppi():
    G, id_map = toy_graph()
    it1, it2 = two_phase_iterators(G, id_map)
    n = len(id_map)
    is_train = np.zeros(n, bool)
    for u in G.nodes():
        is_train[id_map[u]] = not G.node[u]["val"] and not G.node[u]["test"]
    assert it1.deg.shape == (n,) and (it1.deg[~is_train] == 0).all()          # val/test ids are never negatives
    assert on2v.unique_support(it1.deg) >= 20
    seen = 0
    while not it1.end():
        f = it1.next_minibatch_feed_dict()
        b1, b2 = np.array(f["batch1"]), np.array(f["batch2"])
        assert f["batch_size"] == len(b1) == len(b2) and 1 <= len(b1) <= 512
        assert is_train[b1].all() and is_train[b2].all()
        seen += len(b1)
    assert seen == len(it1.train_edges) and seen % 512 != 0                  # the last batch is short
    assert len(it2.train_edges) > 0
    while not it2.end():
        f = it2.next_minibatch_feed_dict()
        b1, b2 = np.array(f["batch1"]), np.array(f["batch2"])
        assert (~is_train[b1]).all() and is_train[b2].all()                  # walks from val/test nodes into the train graph
    # dict_size = N + 1 rows (the trainer's features.shape[0]); negatives are drawn from the N degrees
    check_unique_sample_size(it1.deg, 20)
