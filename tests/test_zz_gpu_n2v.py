"""Node2Vec / DeepWalk baseline on the GPU (reference graphsage/models.py:408-501): gs_sample_unigram_unique bit for bit
against the oracle's sequential rejection loop, gs_skipgram_grad against the oracle and fp64 torch autograd,
gs_embedding_sgd against fp64 index_add_, and Node2VecModel end to end (tracking a CPU restatement, reproducibility,
loss() without update, export, the two-phase flow on the toy-ppi slice)."""
import numpy as np
import pytest
import torch

from graphsage_b200 import ops
from graphsage_b200.node2vec import Node2VecModel, UniqueUnigramSampler
from oracle import node2vec as on2v

pytestmark = pytest.mark.gpu


def _hub(n=50, hub=1e6):
    deg = np.ones(n)
    deg[7] = hub
    deg[3] = 0.0
    return deg


# ------------------------------------------------------------------ gs_sample_unigram_unique
@pytest.mark.parametrize("deg, S", [(np.arange(1, 300, dtype=np.float64), 20), (np.arange(1, 300, dtype=np.float64), 299),
                                    (np.arange(1, 5000, dtype=np.float64) ** 1.5, 1024), (_hub(), 20), (_hub(), 49),
                                    (np.r_[np.zeros(5), np.ones(3)], 3)])
def test_unique_sampler_bit_exact(deg, S):
    cdf = torch.from_numpy(on2v.unigram_cdf(deg)).cuda()
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    for seed, counter in ((123, 0), (123, 1), (9, 1 << 40)):
        got = ops.sample_unigram_unique(cdf, S, seed, counter, status=status).cpu().numpy()
        assert np.array_equal(got, on2v.sample_unigram_unique(deg, S, seed, counter))
    # the device-side counter is added to the host one
    cdev = torch.tensor([5], dtype=torch.int64, device="cuda")
    got = ops.sample_unigram_unique(cdf, S, 123, 2, counter_dev=cdev).cpu().numpy()
    assert np.array_equal(got, on2v.sample_unigram_unique(deg, S, 123, 7))
    assert int(status.item()) == 0


def test_unique_sampler_budget_is_reported():
    deg = np.r_[1e15, 1.0]                                 # id 1 lies below the draws' resolution: never drawn
    cdf = torch.from_numpy(on2v.unigram_cdf(deg)).cuda()
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    got = ops.sample_unigram_unique(cdf, 2, 5, 0, status=status).cpu().numpy()
    assert got.tolist() == [0, -1] and int(status.item()) == 1
    assert np.array_equal(got, on2v.sample_unigram_unique(deg, 2, 5, 0))
    s = UniqueUnigramSampler(deg, 2, device="cuda")
    s()
    with pytest.raises(RuntimeError):
        s.check()


def test_unique_sampler_refusals():
    cdf = torch.from_numpy(on2v.unigram_cdf(np.ones(2000))).cuda()
    with pytest.raises(ValueError):
        ops.sample_unigram_unique(cdf, 1025, 1, 0)
    with pytest.raises(RuntimeError):
        ops.sample_unigram_unique(cdf.cpu(), 4, 1, 0)
    with pytest.raises(ValueError):
        UniqueUnigramSampler(np.r_[np.zeros(5), np.ones(3)], 4, device="cuda")


# ------------------------------------------------------------------ gs_skipgram_grad
def _problem(V, d, B, S, seed, pad=3):
    r = np.random.RandomState(seed)
    T = r.uniform(-1, 1, size=(V, d)).astype(np.float32)
    C = (r.randn(V, d) / np.sqrt(d)).astype(np.float32)
    b = (r.randn(V) * 0.3).astype(np.float32)
    neg = r.choice(V, size=S, replace=False).astype(np.int32)
    b1 = r.randint(0, V, size=B).astype(np.int32)
    b2 = r.randint(0, V, size=B).astype(np.int32)
    b1[1] = b1[0]
    b2[2] = b2[3] = b2[4]
    b2[5] = neg[0]
    # device tables with padded row strides: target [V, d] view, context [V, d + 1] with the bias in column d
    Td = torch.zeros((V, d + pad), device="cuda")
    Td[:, :d] = torch.from_numpy(T).cuda()
    Cd = torch.zeros((V, d + 1 + pad), device="cuda")
    Cd[:, :d] = torch.from_numpy(C).cuda()
    Cd[:, d] = torch.from_numpy(b).cuda()
    return T, C, b, b1, b2, neg, Td[:, :d], Cd[:, :d + 1]


@pytest.mark.parametrize("d", [1, 50, 256])
@pytest.mark.parametrize("B", [512, 37])
def test_skipgram_step_vs_oracle_and_fp64_autograd(d, B):
    V, S = 3000, 20
    T, C, b, b1, b2, neg, Td, Cd = _problem(V, d, B, S, seed=d * 1000 + B)
    dev = lambda x: torch.from_numpy(x).cuda()
    out = ops.skipgram_grad(Td, Cd, dev(b1), dev(b2), dev(neg))
    loss, aff, neg_aff = on2v.skipgram_forward(T, C, b, b1, b2, neg)
    assert abs(out["loss"].item() - loss) <= 2e-5 * abs(loss)
    assert np.allclose(out["aff"].cpu().numpy(), aff, rtol=1e-4, atol=1e-5)
    assert np.allclose(out["neg_aff"].cpu().numpy(), neg_aff, rtol=1e-4, atol=1e-5)
    # fp64 torch autograd on the looked-up rows
    T64, C64, b64 = (torch.from_numpy(x.astype(np.float64)) for x in (T, C, b))
    i1, i2, ineg = (torch.from_numpy(x.astype(np.int64)) for x in (b1, b2, neg))
    t, c, n = T64[i1].requires_grad_(), C64[i2].requires_grad_(), C64[ineg].requires_grad_()
    cb, nb = b64[i2].requires_grad_(), b64[ineg].requires_grad_()
    ref = (torch.nn.functional.softplus(-((t * c).sum(1) + cb)).sum()
           + torch.nn.functional.softplus(t @ n.t() + nb[None, :]).sum()) / B
    ref.backward()
    gc_pos, gc_neg = out["gc_pos"].cpu().double(), out["gc_neg"].cpu().double()
    for got, want in ((out["gt"].cpu().double(), t.grad), (gc_pos[:, :d], c.grad), (gc_pos[:, d], cb.grad),
                      (gc_neg[:, :d], n.grad), (gc_neg[:, d], nb.grad)):
        scale = float(want.abs().max())
        assert float((got - want).abs().max()) <= 1e-5 * scale + 1e-9, (d, B)
    # bit-identical on every call
    again = ops.skipgram_grad(Td, Cd, dev(b1), dev(b2), dev(neg))
    for k in out:
        assert torch.equal(out[k], again[k]), k


def test_skipgram_refusals():
    _, _, _, b1, b2, neg, Td, Cd = _problem(100, 8, 16, 4, seed=1)
    dev = lambda x: torch.from_numpy(x).cuda()
    with pytest.raises(RuntimeError):
        ops.skipgram_grad(Td.cpu(), Cd.cpu(), torch.from_numpy(b1), torch.from_numpy(b2), torch.from_numpy(neg))
    with pytest.raises(ValueError):
        ops.skipgram_grad(Td.double(), Cd.double(), dev(b1), dev(b2), dev(neg))
    with pytest.raises(ValueError):
        ops.skipgram_grad(Td, Cd[:, :8], dev(b1), dev(b2), dev(neg))                # no bias column
    with pytest.raises(ValueError):
        ops.skipgram_grad(Td, Cd, dev(b1), dev(b2[:5]), dev(neg))


# ------------------------------------------------------------------ gs_embedding_sgd
@pytest.mark.parametrize("d", [1, 37, 257])
def test_embedding_sgd_vs_fp64_index_add(d):
    V, lr = 5000, 0.25
    r = np.random.RandomState(d)
    full = torch.from_numpy(r.randn(V, d + 5).astype(np.float32)).cuda()
    table = full[:, :d]
    ids1 = r.randint(0, V, size=700).astype(np.int32)
    ids1[:5000 % 700] = 3
    ids2 = np.r_[np.full(4000, 11, np.int32), r.randint(0, 50, size=300).astype(np.int32)]   # a long run crosses chunks
    g1 = torch.from_numpy(r.randn(700, d + 2).astype(np.float32)).cuda()
    g2 = torch.from_numpy(r.randn(len(ids2), d).astype(np.float32)).cuda()
    lists = [(torch.from_numpy(ids1).cuda(), g1, 1, 1.0), (torch.from_numpy(ids2).cuda(), g2, 1, 0.5)]
    before = full.clone()
    ops.embedding_sgd(table, lists, lr)
    want = before.double().cpu()
    want[:, :d].index_add_(0, torch.from_numpy(ids1).long(), g1[:, :d].double().cpu(), alpha=-lr)
    want[:, :d].index_add_(0, torch.from_numpy(ids2).long(), 0.5 * g2.double().cpu(), alpha=-lr)
    got = full.double().cpu()
    err = (got - want).abs().max().item()
    assert err <= 1e-5 * max(1.0, want.abs().max().item()), err
    touched = np.zeros(V, bool)
    touched[ids1] = touched[ids2] = True
    assert torch.equal(full[torch.from_numpy(~touched).cuda()], before[torch.from_numpy(~touched).cuda()])
    assert torch.equal(full[:, d:], before[:, d:])                          # columns past d are never written
    # bit-identical on every call
    again = before.clone()
    ops.embedding_sgd(again[:, :d], lists, lr)
    assert torch.equal(again, full)


# ------------------------------------------------------------------ Node2VecModel
def _model(seed=3, V=600, d=24, S=10, lr=0.05):
    deg = np.random.RandomState(0).randint(0, 9, size=V - 1).astype(np.float64)      # N degrees, N + 1 rows
    return Node2VecModel({"batch_size": 64}, V, deg, nodevec_dim=d, lr=lr, neg_sample_size=S, seed=seed), deg


def _pairs(V, B, seed):
    r = np.random.RandomState(seed)
    b1, b2 = r.randint(0, V - 1, size=B).astype(np.int32), r.randint(0, V - 1, size=B).astype(np.int32)
    b1[:4] = b1[4]
    b2[:3] = b2[3]
    return b1, b2


def test_model_tracks_cpu_restatement():
    m, deg = _model()
    V, d, lr = 600, 24, 0.05
    assert m.target_embeds.shape == (V, d) and m.context_embeds.shape == (V, d) and m.context_bias.shape == (V,)
    assert float(m.target_embeds.abs().max()) <= 1.0 and float(m.context_bias.abs().max()) == 0.0
    assert float(m.context_embeds.abs().max()) <= 2.0 / np.sqrt(d) + 1e-6
    T = m.target_embeds.double().cpu().numpy()
    C = m.context_embeds.double().cpu().numpy()
    b = m.context_bias.double().cpu().numpy()
    for step in range(6):
        b1, b2 = _pairs(V, 64 if step < 5 else 23, step)
        loss = m.train_step(torch.from_numpy(b1).cuda(), torch.from_numpy(b2).cuda())
        neg = m.neg_samples.cpu().numpy()
        assert np.array_equal(neg, on2v.sample_unigram_unique(deg, 10, 3, step))
        T, C, b, ref_loss = on2v.sgd_step(T, C, b, b1, b2, neg, lr)
        assert abs(loss.item() - ref_loss) <= 1e-5 * abs(ref_loss)
    for got, want in ((m.target_embeds, T), (m.context_embeds, C), (m.context_bias, b)):
        assert np.abs(got.double().cpu().numpy() - want).max() <= 1e-5
    m.neg_sampler.check()


def test_model_reproducible_and_loss_does_not_update():
    runs = []
    for _ in range(2):
        m, _ = _model(seed=11)
        for step in range(4):
            m.train_step(*_pairs(600, 64, step))
        runs.append([x.clone() for x in (m.target_embeds, m.context_embeds, m.context_bias)])
    for a, b in zip(*runs):
        assert torch.equal(a, b)
    m, _ = _model(seed=11)
    before = [x.clone() for x in (m._target, m._context)]
    l1 = m.loss(*_pairs(600, 64, 0))
    mrr = float(m.mrr())
    assert 0.0 < mrr <= 1.0 and l1.dim() == 0
    for a, b in zip(before, (m._target, m._context)):
        assert torch.equal(a, b)
    assert m.neg_sampler.counter == 1                      # every loss evaluation draws fresh negatives


def test_export_writes_the_reference_format(tmp_path):
    m, _ = _model()
    ids = np.arange(0, 599, 3)
    emb = m.export_embeddings(ids, batch_size=50, out_prefix=str(tmp_path / "val"))
    assert emb.shape == (len(ids), 24) and emb.dtype == np.float32
    assert np.array_equal(np.load(str(tmp_path / "val.npy")), emb)
    assert np.array_equal(emb, m.target_embeds.cpu().numpy()[ids])             # outputs1 = target_embeds[batch1]
    assert open(str(tmp_path / "val.txt")).read().split("\n") == [str(i) for i in ids]


def test_two_phase_training_on_toy_ppi():
    from test_n2v_cpu import toy_graph, two_phase_iterators
    G, id_map = toy_graph()
    it1, it2 = two_phase_iterators(G, id_map, batch_size=128)
    n = len(id_map)
    m = Node2VecModel({}, n + 1, it1.deg, nodevec_dim=32, lr=0.5, neg_sample_size=20, seed=4)

    def mean_loss(it, train):
        it.shuffle()
        losses = []
        while not it.end():
            f = it.next_minibatch_feed_dict()
            losses.append((m.train_step if train else m.loss)(f["batch1"], f["batch2"]))
        return float(torch.stack(losses).mean())

    first = mean_loss(it1, False)
    for _ in range(4):
        mean_loss(it1, True)
    after = mean_loss(it1, False)
    assert after < first, (first, after)
    # phase 2: retrain on the val/test walk pairs (all three tables keep training, as the reference effectively does)
    first2 = mean_loss(it2, False)
    for _ in range(4):
        mean_loss(it2, True)
    assert mean_loss(it2, False) < first2
    m.neg_sampler.check()
