"""GPU: minibatches over whole neighbourhoods.  ops.csr_blocks bit for bit against oracle/full_neighbor_blocks.py;
full_neighbor_minibatch_embeddings torch.equal to full_neighbor_embeddings over every aggregator, concat, math, table and
identity_dim; the supervised and unsupervised minibatch losses equal to the whole-graph ones and their gradients close;
Adam steps, determinism, a memory bound against the whole-graph step, a toy-ppi epoch and the refusals."""
import numpy as np
import pytest
import torch

from conftest import load_golden, rel_err
from oracle import full_neighbor_blocks as fb
from test_zz_gpu_full_neighbor import dev, edge_csr, oracle_aggs  # noqa: F401
from test_zz_gpu_full_neighbor_train import POOL_BIAS_TOL, named_grads, sup_model

pytestmark = pytest.mark.gpu
GRAD_TOL = 2e-4


@pytest.fixture(scope="module")
def gs():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    import graphsage_b200
    graphsage_b200._lib.lib()
    return graphsage_b200


# ---------------------------------------------------------------- the block builder, bit for bit
def _graph(case):
    rs = np.random.RandomState(1)
    if case == "empty":
        return np.zeros(51, np.int64), np.zeros(0, np.int32)
    if case == "hub":                                  # a row of 10^5 entries and an in-degree hub (node 3)
        n = 3000
        deg = rs.randint(0, 6, size=n)
        deg[5] = 100000
        indptr = np.concatenate([[0], np.cumsum(deg)]).astype(np.int64)
        indices = rs.randint(-2, n + 2, size=int(indptr[-1])).astype(np.int32)
        indices[::3] = 3
        return indptr, indices
    return edge_csr(rs, 2000, 2000)


def _seeds(case, N):
    rs = np.random.RandomState(2)
    return {"mixed": np.array([5, 5, -1, N, N + 7, 0, 3, 1999 % N, 2], np.int32),
            "random": rs.randint(0, N, size=300).astype(np.int32), "single": np.array([5], np.int32),
            "every node": np.arange(N, dtype=np.int32), "none": np.zeros(0, np.int32)}[case]


@pytest.mark.parametrize("L", [1, 2, 3])
@pytest.mark.parametrize("seeds", ["mixed", "random", "single", "every node", "none"])
@pytest.mark.parametrize("case", ["messy", "hub", "empty"])
def test_csr_blocks_bit_exact(gs, case, seeds, L):
    indptr, indices = _graph(case)
    s = _seeds(seeds, len(indptr) - 1)
    got = gs.ops.csr_blocks(dev(indptr), dev(indices), dev(s), L)
    want = fb.csr_blocks(indptr, indices, s, L)
    assert len(got) == L
    for l, (g, w) in enumerate(zip(got, want)):
        for k in ("src_ids", "indptr", "indices", "rows"):
            t = getattr(g, k)
            assert t.dtype == (torch.int64 if k == "indptr" else torch.int32)
            assert np.array_equal(t.cpu().numpy(), w[k]), (l, k)
    again = gs.ops.csr_blocks(dev(indptr), dev(indices), dev(s), L)
    assert all(torch.equal(a, b) for ga, gb in zip(got, again) for a, b in zip(ga, gb))


def test_csr_blocks_input_checks(gs):
    indptr, indices = _graph("messy")
    with pytest.raises(TypeError, match="indptr"):
        gs.ops.csr_blocks(dev(indptr.astype(np.int32)), dev(indices), dev(np.zeros(1, np.int32)), 2)
    with pytest.raises(TypeError, match="indices"):
        gs.ops.csr_blocks(dev(indptr), dev(indices.astype(np.int64)), dev(np.zeros(1, np.int32)), 2)
    with pytest.raises(TypeError, match="seeds"):
        gs.ops.csr_blocks(dev(indptr), dev(indices), dev(np.zeros(1, np.int64)), 2)
    for L in (0, 9):
        with pytest.raises(ValueError, match="n_layers"):
            gs.ops.csr_blocks(dev(indptr), dev(indices), dev(np.zeros(1, np.int32)), L)
    with pytest.raises(RuntimeError, match="CUDA-only"):
        gs.ops.csr_blocks(torch.from_numpy(indptr), dev(indices), dev(np.zeros(1, np.int32)), 2)


# ---------------------------------------------------------------- inference: the same bits as the whole graph
def emb_model(gs, kind, concat, math, variant, layers, n=300, F=20, seed=0):
    """variant: the layer-0 table - "fp32", "bf16", "fp32+16" (identity_dim 16 in front of fp32 features) or "none+16"
    (identity_dim 16, no feature table)."""
    rs = np.random.RandomState(seed)
    feats = np.vstack([rs.randn(n, F).astype(np.float32), np.zeros((1, F), np.float32)])
    gs.set_default_math(math)
    gs.inits.manual_seed(seed + 1)
    adj = rs.randint(0, n, size=(n + 1, 8)).astype(np.int32)
    adj[n] = n
    adj = dev(adj)
    sampler = gs.UniformNeighborSampler(adj, seed=3)
    infos = [gs.SAGEInfo("node", sampler, 5, d) for d in [16, 12, 8][:layers]]
    f = None if variant == "none+16" else dev(feats).to(torch.bfloat16) if variant == "bf16" else dev(feats)
    m = gs.SampleAndAggregate({"batch_size": 8, "dropout": 0.}, f, adj, None, infos, concat=concat, aggregator_type=kind,
                              identity_dim=16 if variant.endswith("+16") else 0)
    gs.set_default_math("fp32")
    return m


@pytest.mark.parametrize("variant", ["fp32", "bf16", "fp32+16", "none+16"])
@pytest.mark.parametrize("math", ["fp32", "tf32x3"])
@pytest.mark.parametrize("kind,concat", [(k, c) for k in ("mean", "maxpool", "meanpool") for c in (False, True)]
                         + [("gcn", False)])          # GCN with concat off, as in the whole-graph tests
def test_minibatch_embeddings_equal_the_whole_graph(gs, kind, concat, math, variant):
    indptr, indices = (dev(a) for a in edge_csr(np.random.RandomState(1), 300, 300))
    for layers in (1, 2, 3):
        m = emb_model(gs, kind, concat, math, variant, layers)
        for ids in (np.array([0, 5, 299, 17, 17, 4, 150, 300, -3, 6], np.int32), np.array([42], np.int32),
                    np.arange(300, dtype=np.int32)):
            for normalize in (True, False):
                want = m.full_neighbor_embeddings(indptr, indices, ids, normalize=normalize)
                got = m.full_neighbor_minibatch_embeddings(indptr, indices, ids, normalize=normalize)
                assert torch.equal(got, want), (layers, len(ids), normalize, (got - want).abs().max())


# ---------------------------------------------------------------- supervised training
def _whole_and_block(m, indptr, indices, ids, labels):
    """(loss, grads) of the whole-graph and of the minibatch loss at the same parameters."""
    out = []
    for fn in (m.full_neighbor_loss, m.full_neighbor_minibatch_loss):
        m.optimizer.zero_grad(set_to_none=True)
        loss = fn(indptr, indices, ids, labels)
        loss.backward()
        out.append((loss.detach(), {k: v.grad.clone() for k, v in named_grads(m) if v.grad is not None},
                    None if m.embeds is None else m.embeds.grad.clone()))
    return out


def check_close(whole, block):
    assert set(whole[1]) == set(block[1])
    for k, g in whole[1].items():
        tol = POOL_BIAS_TOL if k[1] == "mlp_bias" else GRAD_TOL
        assert rel_err(block[1][k].cpu().numpy(), g.cpu().numpy()) < tol, k
    if whole[2] is not None:
        assert rel_err(block[2].cpu().numpy(), whole[2].cpu().numpy()) < GRAD_TOL


SUP_CASES = ([(k, c, "fp32", "fp32", 0, 2) for k in ("mean", "maxpool", "meanpool") for c in (False, True)]
             + [("gcn", False, "fp32", "fp32", 0, 2), ("mean", True, "tf32x3", "fp32", 0, 2),
                ("maxpool", True, "tf32x3", "fp32", 0, 2), ("maxpool", False, "fp32", "bf16", 0, 2),
                ("meanpool", True, "fp32", "bf16", 0, 2), ("mean", True, "fp32", "fp32", 16, 2),
                ("maxpool", True, "fp32", "fp32", 16, 2), ("gcn", False, "tf32x3", "fp32", 16, 2),
                ("meanpool", False, "fp32", "fp32", 16, 1), ("mean", True, "fp32", "fp32", 0, 3),
                ("maxpool", True, "tf32x3", "fp32", 16, 3), ("gcn", False, "fp32", "fp32", 16, 3)])


@pytest.mark.parametrize("kind,concat,math,table,identity_dim,layers", SUP_CASES)
def test_supervised_loss_and_gradients_match_the_whole_graph(gs, kind, concat, math, table, identity_dim, layers):
    m = sup_model(gs, kind, concat, math, table, identity_dim, layers, sigmoid=layers == 3)
    indptr, indices = (dev(a) for a in edge_csr(np.random.RandomState(1), 300, 300))
    ids = np.array([0, 5, 299, 17, 17, 4, 150, 6, 1, 2, 3, -1], dtype=np.int32)
    labels = np.eye(4, dtype=np.float32)[np.arange(len(ids)) % 4]
    assert torch.equal(m.full_neighbor_minibatch_outputs(indptr, indices, ids).detach(),
                       m.full_neighbor_outputs(indptr, indices, ids).detach())
    whole, block = _whole_and_block(m, indptr, indices, ids, labels)
    assert torch.equal(block[0], whole[0])
    check_close(whole, block)


@pytest.mark.parametrize("kind", ["mean", "maxpool"])
def test_five_adam_steps_track_the_whole_graph_steps(gs, kind):
    indptr, indices = (dev(a) for a in edge_csr(np.random.RandomState(2), 300, 300))
    ids = np.arange(0, 300, 7, dtype=np.int32)
    labels = np.eye(4, dtype=np.float32)[ids % 4]
    runs = []
    for step in ("full_neighbor_train_step", "full_neighbor_minibatch_train_step"):
        m = sup_model(gs, kind, identity_dim=8)
        losses = [float(getattr(m, step)(indptr, indices, ids, labels)) for _ in range(5)]
        runs.append((losses, [p.detach().cpu().numpy() for p in m.parameters()]))
    assert np.allclose(runs[0][0], runs[1][0], rtol=1e-4)
    for a, b in zip(runs[0][1], runs[1][1]):   # Adam's normalised step amplifies differences in near-zero gradients
        assert rel_err(b, a) < 1e-2


@pytest.mark.parametrize("kind", ["mean", "maxpool"])
def test_two_steps_from_the_same_state_are_bit_identical(gs, kind):
    indptr, indices = (dev(a) for a in edge_csr(np.random.RandomState(3), 300, 300))
    ids = np.arange(0, 300, 5, dtype=np.int32)
    labels = np.eye(4, dtype=np.float32)[ids % 4]
    runs = []
    for _ in range(2):
        m = sup_model(gs, kind, identity_dim=8)
        losses = [m.full_neighbor_minibatch_train_step(indptr, indices, ids, labels) for _ in range(2)]
        runs.append((losses, [p.detach().clone() for p in m.parameters()]))
    assert all(torch.equal(a, b) for a, b in zip(runs[0][0], runs[1][0]))
    assert all(torch.equal(a, b) for a, b in zip(runs[0][1], runs[1][1]))


# ---------------------------------------------------------------- unsupervised training
def unsup_model(gs, kind, identity_dim=0, n=300, F=20):
    rs = np.random.RandomState(0)
    feats = np.vstack([rs.randn(n, F).astype(np.float32), np.zeros((1, F), np.float32)])
    gs.inits.manual_seed(1)
    adj = rs.randint(0, n, size=(n + 1, 8)).astype(np.int32)
    adj[n] = n
    adj = dev(adj)
    sampler = gs.UniformNeighborSampler(adj, seed=3)
    infos = [gs.SAGEInfo("node", sampler, 5, d) for d in (16, 12)]
    return gs.UnsupervisedGraphsage({"batch_size": 8, "dropout": 0.}, dev(feats), adj, rs.randint(1, 9, size=n), infos,
                                    concat=kind != "gcn", aggregator_type=kind, identity_dim=identity_dim,
                                    neg_sample_size=6, weight_decay=0.01, learning_rate=0.01)


@pytest.mark.parametrize("kind,identity_dim", [("mean", 0), ("gcn", 16), ("maxpool", 16), ("meanpool", 0)])
def test_unsupervised_loss_and_gradients_match_the_whole_graph(gs, kind, identity_dim):
    from graphsage_b200.full_neighbor_training import full_neighbor_outputs
    from graphsage_b200.supervised_models import weight_decay_term
    m = unsup_model(gs, kind, identity_dim)
    indptr, indices = (dev(a) for a in edge_csr(np.random.RandomState(4), 300, 300))
    b1 = torch.tensor([0, 5, 17, 17, 299, 6], dtype=torch.int32)
    b2 = torch.tensor([1, 1, 40, 250, 3, 6], dtype=torch.int32)
    c0 = m.neg_sampler.counter
    loss = m.full_neighbor_minibatch_loss(indptr, indices, b1, b2)
    assert m.neg_sampler.counter == c0 + 1
    loss.backward()
    got = {id(p): p.grad.clone() for p in m.parameters() if p.grad is not None}
    mrr = float(m.mrr())
    assert np.isfinite(mrr)
    m.neg_sampler.counter = c0                                           # the same negatives
    neg = m.neg_sampler(m.neg_sample_size)
    m.optimizer.zero_grad(set_to_none=True)
    out = full_neighbor_outputs(m, indptr, indices, torch.cat([b1.cuda(), b2.cuda(), neg]))
    o1, o2, on = torch.split(out, [6, 6, neg.numel()])
    want = (m.link_pred_layer.loss(o1, o2, on) + weight_decay_term(m.decayed_parameters(), m.weight_decay)) / 6.0
    want.backward()
    assert torch.equal(loss.detach(), want.detach())
    assert set(got) == {id(p) for p in m.parameters() if p.grad is not None}
    names = {id(v): k for k, v in named_grads_unsup(m)}
    for p in m.parameters():
        if p.grad is not None:
            tol = POOL_BIAS_TOL if names.get(id(p)) == "mlp_bias" else GRAD_TOL
            assert rel_err(got[id(p)].cpu().numpy(), p.grad.cpu().numpy()) < tol, names.get(id(p))
    c1 = m.neg_sampler.counter
    for _ in range(2):
        m.full_neighbor_minibatch_train_step(indptr, indices, b1, b2)
    assert m.neg_sampler.counter == c1 + 2 and np.isfinite(float(m.mrr()))


def named_grads_unsup(m):
    out = []
    for a in m.aggregators:
        out += list(a.vars.items())
        if hasattr(a, "mlp_layers"):
            out += [("mlp_weights", a.mlp_layers[0].vars["weights"]), ("mlp_bias", a.mlp_layers[0].vars["bias"])]
    return out


# ---------------------------------------------------------------- memory, toy-ppi, refusals
def test_peak_memory_is_a_fraction_of_the_whole_graph_step(gs):
    n, F = 200000, 64
    rs = np.random.RandomState(5)
    deg = rs.randint(1, 8, size=n)                                         # mean degree 4
    indptr = np.concatenate([[0], np.cumsum(deg)]).astype(np.int64)
    indices = rs.randint(0, n, size=int(indptr[-1])).astype(np.int32)
    m = sup_model(gs, "mean", n=n, F=F, adj=np.full((n + 1, 8), n, np.int32))
    ids = rs.randint(0, n, size=256).astype(np.int32)
    labels = dev(np.eye(4, dtype=np.float32)[ids % 4])
    d_indptr, d_indices, d_ids = dev(indptr), dev(indices), dev(ids)
    peaks = []
    for step in (m.full_neighbor_train_step, m.full_neighbor_minibatch_train_step):
        step(d_indptr, d_indices, d_ids, labels)                          # transposes cached, Adam state allocated
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        step(d_indptr, d_indices, d_ids, labels)
        torch.cuda.synchronize()
        peaks.append(torch.cuda.max_memory_allocated() - base)
    print("peak MB: whole graph %.1f, minibatch %.1f" % (peaks[0] / 2**20, peaks[1] / 2**20))
    assert peaks[1] * 4 < peaks[0], peaks


def test_toy_ppi_minibatch_epoch(gs):
    from test_walks_cpu import toy_graph
    from graphsage_b200.minibatch import NodeMinibatchIterator
    from graphsage_b200.supervised_train import calc_f1
    g = load_golden("toy_ppi")
    G = toy_graph()
    id2idx = {u: i for i, u in enumerate(G.nodes())}
    labels = (np.asarray(g["labels"]) > 0).astype(np.float32)
    it = NodeMinibatchIterator(G, id2idx, None, {u: labels[i] for i, u in enumerate(G.nodes())}, labels.shape[1],
                               batch_size=64, max_degree=25, rng=np.random.RandomState(0))
    n = len(id2idx)
    feats = torch.zeros((n + 1, 50), device="cuda")
    feats[:n] = dev(np.asarray(g["feats"], np.float32))
    gs.inits.manual_seed(3)
    sampler = gs.UniformNeighborSampler(dev(it.adj), seed=1)
    infos = [gs.SAGEInfo("node", sampler, 10, 64), gs.SAGEInfo("node", sampler, 5, 64)]
    m = gs.SupervisedGraphsage(labels.shape[1], {"batch_size": 512, "dropout": 0.}, feats, dev(it.adj), None, infos,
                               aggregator_type="mean", sigmoid_loss=True, learning_rate=0.03)
    train = np.array([id2idx[u] for u in G.nodes() if not G.node[u]["val"] and not G.node[u]["test"]], dtype=np.int32)
    val = np.array([id2idx[u] for u in G.nodes() if G.node[u]["val"]], dtype=np.int32)
    tr_ptr, tr_idx = (dev(a) for a in it.neighbor_csr(test=False))
    te_ptr, te_idx = it.neighbor_csr(test=True)
    d_lab = dev(labels)

    def train_loss():
        with torch.no_grad():
            return float(m.full_neighbor_minibatch_loss(tr_ptr, tr_idx, train, d_lab[train]))
    before = calc_f1(labels[val], m.full_neighbor_predict(te_ptr, te_idx, val).cpu().numpy(), True)[0], train_loss()
    order = np.random.RandomState(0).permutation(train)
    steps = 0
    for i in range(0, len(order), 512):
        b = dev(order[i:i + 512])
        m.full_neighbor_minibatch_train_step(tr_ptr, tr_idx, b, d_lab[b.long()])
        steps += 1
    after = calc_f1(labels[val], m.full_neighbor_predict(te_ptr, te_idx, val).cpu().numpy(), True)[0], train_loss()
    print("toy-ppi minibatch epoch (%d steps of 512): train loss %.4f -> %.4f, val F1 micro %.4f -> %.4f"
          % (steps, before[1], after[1], before[0], after[0]))
    assert after[1] < before[1]
    assert after[0] > before[0]


def test_refusals(gs, monkeypatch):
    indptr, indices = edge_csr(np.random.RandomState(0), 300, 300)
    ids, labels = np.arange(4, dtype=np.int32), np.eye(4, dtype=np.float32)
    m = sup_model(gs, "mean")
    m.dropout_rate = 0.5
    with pytest.raises(NotImplementedError, match="dropout"):
        m.full_neighbor_minibatch_train_step(indptr, indices, ids, labels)
    m.dropout_rate = 0.
    with pytest.raises(ValueError, match="N \\+ 1"):
        m.full_neighbor_minibatch_loss(indptr[:-1], indices, ids, labels)
    with pytest.raises(TypeError, match="indices"):
        m.full_neighbor_minibatch_embeddings(indptr, indices.astype(np.int64), ids)
    monkeypatch.setattr(torch.cuda, "is_current_stream_capturing", lambda: True)
    with pytest.raises(NotImplementedError, match="CUDA graph"):
        m.full_neighbor_minibatch_train_step(indptr, indices, ids, labels)
    with pytest.raises(NotImplementedError, match="CUDA graph"):
        m.full_neighbor_minibatch_embeddings(indptr, indices, ids)
    u = unsup_model(gs, "mean")
    c0 = u.neg_sampler.counter
    with pytest.raises(NotImplementedError, match="CUDA graph"):
        u.full_neighbor_minibatch_train_step(indptr, indices, ids, ids)
    assert u.neg_sampler.counter == c0
