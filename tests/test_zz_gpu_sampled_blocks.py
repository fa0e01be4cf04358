"""GPU: minibatches over sampled neighbourhoods.  ops.csr_blocks(..., fanouts) and ops.sample_csr_rows byte for byte
against oracle/sampled_blocks.py; with every fanout >= the largest degree the blocks, embeddings, losses and gradients
equal the whole-neighbourhood minibatch ones; one layer equals full_neighbor_embeddings over the sample; losses and
gradients against the CPU oracle; determinism, a memory bound on a hub-heavy graph, a toy-ppi epoch and the refusals."""
import numpy as np
import pytest
import torch

from conftest import load_golden, rel_err
from oracle import rmat
from oracle import sampled_blocks as sb
from test_zz_gpu_full_neighbor import dev, edge_csr, oracle_aggs  # noqa: F401
from test_zz_gpu_full_neighbor_minibatch import _graph, emb_model, named_grads_unsup, unsup_model
from test_zz_gpu_full_neighbor_train import POOL_BIAS_TOL, named_grads, sup_model

pytestmark = pytest.mark.gpu
GRAD_TOL = 2e-4


@pytest.fixture(scope="module")
def gs():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    import graphsage_b200
    graphsage_b200._lib.lib()
    return graphsage_b200


def _toy_ppi_csr():
    from test_walks_cpu import toy_graph
    from graphsage_b200.minibatch import NodeMinibatchIterator
    G = toy_graph()
    id2idx = {u: i for i, u in enumerate(G.nodes())}
    it = NodeMinibatchIterator(G, id2idx, None, {u: np.zeros(2) for u in G.nodes()}, 2, batch_size=64, max_degree=25,
                               rng=np.random.RandomState(0))
    return it.neighbor_csr(test=False)


def _rmat_csr(scale=14):
    """A hub-heavy R-MAT graph (mean degree 12) with one extra row of 10^5 entries (node 17)."""
    indptr, indices = rmat.rmat_csr(scale, 1 << scale, edge_factor=12.0, seed=4)
    hub = np.random.RandomState(6).randint(0, 1 << scale, size=100000).astype(np.int32)
    v = 17
    indices = np.concatenate([indices[:indptr[v + 1]], hub, indices[indptr[v + 1]:]]).astype(np.int32)
    indptr = indptr.copy()
    indptr[v + 1:] += len(hub)
    return indptr, indices


GRAPHS = {}


def graph(name):
    if name not in GRAPHS:
        GRAPHS[name] = {"toy-ppi": _toy_ppi_csr, "rmat": _rmat_csr, "messy": lambda: _graph("messy"),
                        "empty": lambda: _graph("empty")}[name]()
    return GRAPHS[name]


def _check_blocks(got, want):
    assert len(got) == len(want)
    for g, w in zip(got, want):
        for key, t in zip(("src_ids", "indptr", "indices", "rows"), g):
            ref = np.asarray(w[key])
            assert t.dtype == (torch.int64 if key == "indptr" else torch.int32)
            assert np.array_equal(t.cpu().numpy(), ref), key


# ---------------------------------------------------------------- the block builder, bit for bit
@pytest.mark.parametrize("k", [1, 10, 25, 256])
@pytest.mark.parametrize("name", ["toy-ppi", "rmat", "messy", "empty"])
def test_sampled_blocks_bit_exact(gs, name, k):
    indptr, indices = graph(name)
    N = len(indptr) - 1
    rs = np.random.RandomState(k)
    seeds = np.concatenate([rs.randint(0, max(N, 1), size=200), [17, 17, -1, N, N + 4]]).astype(np.int32)
    for L in (1, 2, 3):
        fanouts = [k, max(1, k // 2), k][:L]
        for seed, call in ((123, 0), (123, 1), (2**63 + 7, 0), (2**63 + 7, 5)):
            got = gs.ops.csr_blocks(dev(indptr), dev(indices), dev(seeds), L, fanouts=fanouts, seed=seed, call=call)
            _check_blocks(got, sb.sampled_blocks(indptr, indices, seeds, fanouts, seed, call))
            if L == 2 and call == 1:
                again = gs.ops.csr_blocks(dev(indptr), dev(indices), dev(seeds), L, fanouts=fanouts, seed=seed,
                                          call=call)
                assert all(torch.equal(a, b) for x, y in zip(got, again) for a, b in zip(x, y))


@pytest.mark.parametrize("k", [1, 10, 25, 256])
@pytest.mark.parametrize("name", ["toy-ppi", "rmat", "messy", "empty"])
def test_sample_csr_rows_bit_exact(gs, name, k):
    indptr, indices = graph(name)
    for seed, call, layer in ((123, 0, 0), (123, 1, 1), (5, 2**40 + 9, 7)):
        s_ptr, s_idx = gs.ops.sample_csr_rows(dev(indptr), dev(indices), k, seed, call, layer)
        w_ptr, w_idx = sb.sample_rows(indptr, indices, k, seed, call, layer)
        assert s_ptr.dtype == torch.int64 and s_idx.dtype == torch.int32
        assert np.array_equal(s_ptr.cpu().numpy(), w_ptr) and np.array_equal(s_idx.cpu().numpy(), w_idx)


def test_input_checks(gs):
    indptr, indices = (dev(a) for a in graph("messy"))
    ids = dev(np.arange(4, dtype=np.int32))
    for fan in ([0], [257], [3, 3]):
        with pytest.raises(ValueError):
            gs.ops.csr_blocks(indptr, indices, ids, 1, fanouts=fan)
    with pytest.raises(ValueError, match="fanout"):
        gs.ops.sample_csr_rows(indptr, indices, 0, 0, 0, 0)
    with pytest.raises(ValueError, match="layer"):
        gs.ops.sample_csr_rows(indptr, indices, 3, 0, 0, 8)


# ---------------------------------------------------------------- fanouts >= every degree: the whole-neighbourhood blocks
def capped_csr(cap=256):
    indptr, indices = edge_csr(np.random.RandomState(1), 300, 300)
    deg = np.minimum(np.diff(indptr), cap)
    keep = np.concatenate([np.arange(indptr[v], indptr[v] + deg[v]) for v in range(len(deg))])
    return np.concatenate([[0], np.cumsum(deg)]).astype(np.int64), indices[keep]


def _set_fanouts(m, k):
    m.layer_infos = [info._replace(num_samples=k) for info in m.layer_infos]


def test_large_fanouts_give_the_csr_blocks(gs):
    indptr, indices = capped_csr()
    ids = dev(np.array([0, 5, 299, 17, 17, 4, 150, 300, -3, 6], np.int32))
    for L in (1, 2, 3):
        want = gs.ops.csr_blocks(dev(indptr), dev(indices), ids, L)
        got = gs.ops.csr_blocks(dev(indptr), dev(indices), ids, L, fanouts=[256] * L, seed=9, call=2)
        assert all(torch.equal(a, b) for x, y in zip(got, want) for a, b in zip(x, y))


@pytest.mark.parametrize("variant", ["fp32", "bf16", "fp32+16"])
@pytest.mark.parametrize("math", ["fp32", "tf32x3"])
@pytest.mark.parametrize("kind,concat", [(k, c) for k in ("mean", "maxpool", "meanpool") for c in (False, True)]
                         + [("gcn", False)])
def test_large_fanout_embeddings_equal_the_minibatch(gs, kind, concat, math, variant):
    indptr, indices = (dev(a) for a in capped_csr())
    for layers in (1, 2):
        m = emb_model(gs, kind, concat, math, variant, layers)
        _set_fanouts(m, 256)
        for ids in (np.array([0, 5, 299, 17, 17, 4, 150, 300, -3, 6], np.int32), np.arange(300, dtype=np.int32)):
            want = m.full_neighbor_minibatch_embeddings(indptr, indices, ids)
            got = m.sampled_minibatch_embeddings(indptr, indices, ids)
            assert torch.equal(got, want), (layers, len(ids), (got - want).abs().max())


def _grads(m):
    return {k: v.grad.clone() for k, v in named_grads(m) if v.grad is not None}, \
        None if m.embeds is None else m.embeds.grad.clone()


@pytest.mark.parametrize("kind,concat,math,table,identity_dim", [
    ("mean", True, "fp32", "fp32", 0), ("mean", False, "tf32x3", "bf16", 0), ("gcn", False, "fp32", "fp32", 16),
    ("maxpool", True, "tf32x3", "fp32", 16), ("maxpool", False, "fp32", "bf16", 0), ("meanpool", True, "fp32", "fp32", 0),
    ("meanpool", False, "tf32x3", "fp32", 16)])
def test_large_fanout_losses_and_gradients_equal_the_minibatch(gs, kind, concat, math, table, identity_dim):
    m = sup_model(gs, kind, concat, math, table, identity_dim)
    _set_fanouts(m, 256)
    indptr, indices = (dev(a) for a in capped_csr())
    ids = np.array([0, 5, 299, 17, 17, 4, 150, 6, 1, 2, 3, -1], dtype=np.int32)
    labels = np.eye(4, dtype=np.float32)[np.arange(len(ids)) % 4]
    out = []
    for fn in (m.full_neighbor_minibatch_loss, m.sampled_minibatch_loss):
        m.optimizer.zero_grad(set_to_none=True)
        loss = fn(indptr, indices, ids, labels)
        loss.backward()
        out.append((loss.detach(),) + _grads(m))
    assert torch.equal(out[0][0], out[1][0])
    assert set(out[0][1]) == set(out[1][1])
    for k in out[0][1]:
        assert torch.equal(out[0][1][k], out[1][1][k]), k
    assert (out[0][2] is None) == (out[1][2] is None)
    if out[0][2] is not None:
        assert torch.equal(out[0][2], out[1][2])


@pytest.mark.parametrize("kind,concat", [("mean", True), ("gcn", False), ("maxpool", False), ("meanpool", True)])
def test_one_layer_equals_the_whole_graph_over_the_sample(gs, kind, concat):
    indptr, indices = (dev(a) for a in edge_csr(np.random.RandomState(1), 300, 300))
    m = emb_model(gs, kind, concat, "fp32", "fp32", 1)
    sampler = m.layer_infos[0].neigh_sampler
    ids = np.array([0, 5, 299, 17, 17, 4, 150, 300, -3, 6], np.int32)
    call = sampler.counter
    got = m.sampled_minibatch_embeddings(indptr, indices, ids)
    assert sampler.counter == call + 1
    s_ptr, s_idx = gs.ops.sample_csr_rows(indptr, indices, m.layer_infos[0].num_samples, sampler.seed, call, 0)
    assert torch.equal(got, m.full_neighbor_embeddings(s_ptr, s_idx, ids))


# ---------------------------------------------------------------- against the CPU oracle
@pytest.mark.parametrize("kind,concat,math,identity_dim,layers,fanout", [
    ("mean", True, "fp32", 0, 2, 5), ("gcn", False, "fp32", 16, 2, 10), ("maxpool", True, "tf32x3", 0, 2, 3),
    ("meanpool", False, "fp32", 16, 2, 25), ("mean", False, "tf32x3", 16, 3, 4), ("maxpool", False, "fp32", 16, 1, 1)])
def test_supervised_loss_and_gradients_match_the_oracle(gs, kind, concat, math, identity_dim, layers, fanout):
    m = sup_model(gs, kind, concat, math, "fp32", identity_dim, layers, fanout=fanout)
    indptr, indices = edge_csr(np.random.RandomState(1), 300, 300)
    ids = np.array([0, 5, 299, 17, 17, 4, 150, 6, 1, 2, 3, -1], dtype=np.int32)
    labels = np.eye(4, dtype=np.float32)[np.arange(len(ids)) % 4]
    sampler = m.layer_infos[0].neigh_sampler
    call = sampler.counter
    feats = m.features.float().cpu().numpy()
    m.optimizer.zero_grad(set_to_none=True)
    loss = m.sampled_minibatch_loss(dev(indptr), dev(indices), ids, labels)
    loss.backward()
    fanouts = [info.num_samples for info in m.layer_infos]
    rl, grads, head, demb = sb.sampled_loss_grads(feats, indptr, indices, oracle_aggs(m), concat,
                                                  np.where((ids < 0) | (ids >= 300), 300, ids), labels,
                                                  m.node_pred_vars["weights"].detach().cpu().numpy(),
                                                  m.node_pred_vars["bias"].detach().cpu().numpy(), fanouts, sampler.seed,
                                                  call, False, m.weight_decay, identity_dim)
    assert abs(float(loss) - rl) < GRAD_TOL * max(1.0, abs(rl))
    for l, a in enumerate(m.aggregators):
        for k, v in a.vars.items():
            assert rel_err(v.grad.cpu().numpy(), grads[l][k]) < GRAD_TOL, (l, k)
        if hasattr(a, "mlp_layers"):
            assert rel_err(a.mlp_layers[0].vars["weights"].grad.cpu().numpy(), grads[l]["mlp_weights"]) < GRAD_TOL
            assert rel_err(a.mlp_layers[0].vars["bias"].grad.cpu().numpy(), grads[l]["mlp_bias"]) < POOL_BIAS_TOL
    assert rel_err(m.node_pred_vars["weights"].grad.cpu().numpy(), head["weights"]) < GRAD_TOL
    if identity_dim:
        assert rel_err(m.embeds.grad.cpu().numpy(), demb) < GRAD_TOL


@pytest.mark.parametrize("kind,identity_dim", [("mean", 0), ("maxpool", 16)])
def test_unsupervised_loss_matches_one_block_set(gs, kind, identity_dim):
    m = unsup_model(gs, kind, identity_dim)
    indptr, indices = (dev(a) for a in edge_csr(np.random.RandomState(1), 300, 300))
    b1 = dev(np.array([1, 2, 3, 9, 40], np.int32))
    b2 = dev(np.array([4, 4, 38, 0, 299], np.int32))
    sampler = m.layer_infos[0].neigh_sampler
    call, neg_state = sampler.counter, m.neg_sampler.counter
    loss = m.sampled_minibatch_loss(indptr, indices, b1, b2)
    assert sampler.counter == call + 1
    mrr = float(m.mrr())
    loss.backward()
    got = [v.grad.clone() for _, v in named_grads_unsup(m)]
    # again from the same counters: the negatives, then one block set over cat(b1, b2, neg)
    m.neg_sampler.counter, sampler.counter = neg_state, call
    m.optimizer.zero_grad(set_to_none=True)
    neg = m.neg_sampler(m.neg_sample_size)
    from graphsage_b200.full_neighbor_training import full_neighbor_outputs
    out = full_neighbor_outputs(m, indptr, indices, torch.cat([b1, b2, neg]), minibatch=True, sampled=True)
    want = m._pairs_loss(*torch.split(out, [5, 5, neg.numel()]))
    want.backward()
    assert torch.equal(loss.detach(), want.detach()) and float(m.mrr()) == mrr
    for (k, v), g in zip(named_grads_unsup(m), got):
        assert torch.equal(v.grad, g), k


def test_repeated_calls_with_one_counter_are_bit_identical(gs):
    indptr, indices = (dev(a) for a in graph("rmat"))
    ids = dev(np.random.RandomState(0).randint(0, 1 << 14, size=512).astype(np.int32))
    labels = dev(np.eye(4, dtype=np.float32)[np.arange(512) % 4])
    runs = []
    for _ in range(2):
        m = sup_model(gs, "maxpool", n=1 << 14, F=32, fanout=10, adj=np.full(((1 << 14) + 1, 8), 1 << 14, np.int32))
        losses = [m.sampled_minibatch_train_step(indptr, indices, ids, labels) for _ in range(2)]
        runs.append((losses, [p.detach().clone() for p in m.parameters()]))
    assert all(torch.equal(a, b) for a, b in zip(runs[0][0], runs[1][0]))
    assert all(torch.equal(a, b) for a, b in zip(runs[0][1], runs[1][1]))


# ---------------------------------------------------------------- memory, toy-ppi, refusals
def test_peak_memory_on_a_hub_heavy_graph(gs):
    indptr, indices = rmat.rmat_csr(17, 1 << 17, edge_factor=12.0, seed=5)
    n = len(indptr) - 1
    m = sup_model(gs, "mean", n=n, F=128, fanout=5, adj=np.full((n + 1, 8), n, np.int32))
    ids = np.random.RandomState(5).randint(0, n, size=1024).astype(np.int32)
    full = gs.ops.csr_blocks(dev(indptr), dev(indices), dev(ids), 2)
    sampled = gs.ops.csr_blocks(dev(indptr), dev(indices), dev(ids), 2, fanouts=[5, 5], seed=1, call=0)
    print("|V_0|: whole neighbourhoods %d of %d nodes, sampled %d" % (full[0].src_ids.numel(), n,
                                                                      sampled[0].src_ids.numel()))
    active = int((np.diff(indptr) > 0).sum())                            # R-MAT leaves many nodes isolated
    print("nodes with an edge: %d" % active)
    assert full[0].src_ids.numel() > active // 2                         # the whole-neighbourhood field: most of them
    assert sampled[0].src_ids.numel() * 5 < full[0].src_ids.numel()
    labels = dev(np.eye(4, dtype=np.float32)[ids % 4])
    d_indptr, d_indices, d_ids = dev(indptr), dev(indices), dev(ids)
    peaks = []
    for step in (m.full_neighbor_minibatch_train_step, m.sampled_minibatch_train_step):
        step(d_indptr, d_indices, d_ids, labels)
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        step(d_indptr, d_indices, d_ids, labels)
        torch.cuda.synchronize()
        peaks.append(torch.cuda.max_memory_allocated() - base)
    print("peak MB: whole-neighbourhood blocks %.1f, sampled blocks %.1f" % (peaks[0] / 2**20, peaks[1] / 2**20))
    # the sampled step still holds the block builder's O(N) workspace (about 5 MB here), so the ratio is below |V_0|'s
    assert peaks[1] * 2 < peaks[0], peaks


def test_toy_ppi_epoch_matches_the_tree_path(gs):
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
    train = np.array([id2idx[u] for u in G.nodes() if not G.node[u]["val"] and not G.node[u]["test"]], dtype=np.int32)
    val = np.array([id2idx[u] for u in G.nodes() if G.node[u]["val"]], dtype=np.int32)
    tr_ptr, tr_idx = (dev(a) for a in it.neighbor_csr(test=False))
    d_lab = dev(labels)
    order = np.random.RandomState(0).permutation(train)
    f1 = {}
    for path in ("tree", "sampled"):
        gs.inits.manual_seed(3)
        sampler = gs.UniformNeighborSampler(dev(it.adj), seed=1)
        infos = [gs.SAGEInfo("node", sampler, 10, 64), gs.SAGEInfo("node", sampler, 5, 64)]
        m = gs.SupervisedGraphsage(labels.shape[1], {"batch_size": 512, "dropout": 0.}, feats, dev(it.adj), None, infos,
                                   aggregator_type="mean", sigmoid_loss=True, learning_rate=0.03)
        for i in range(0, len(order), 512):
            b = dev(order[i:i + 512])
            if path == "tree":
                m.train_step(b, d_lab[b.long()])
            else:
                m.sampled_minibatch_train_step(tr_ptr, tr_idx, b, d_lab[b.long()])
        sampler.set_adj(dev(it.test_adj))
        with torch.no_grad():
            pred = m.predict(dev(val)).cpu().numpy()
        f1[path] = calc_f1(labels[val], pred, True)[0]
    print("toy-ppi one epoch of 512-node steps: val micro-F1 tree %.4f, sampled blocks %.4f" % (f1["tree"],
                                                                                               f1["sampled"]))
    assert abs(f1["tree"] - f1["sampled"]) <= 0.02


def test_refusals(gs, monkeypatch):
    indptr, indices = edge_csr(np.random.RandomState(0), 300, 300)
    ids, labels = np.arange(4, dtype=np.int32), np.eye(4, dtype=np.float32)
    m = sup_model(gs, "mean")
    sampler = m.layer_infos[0].neigh_sampler
    m.dropout_rate = 0.5
    with pytest.raises(NotImplementedError, match="dropout"):
        m.sampled_minibatch_train_step(indptr, indices, ids, labels)
    m.dropout_rate = 0.
    with pytest.raises(ValueError, match="N \\+ 1"):
        m.sampled_minibatch_loss(indptr[:-1], indices, ids, labels)
    _set_fanouts(m, 300)
    with pytest.raises(ValueError, match="fanout"):
        m.sampled_minibatch_loss(indptr, indices, ids, labels)
    assert sampler.counter == 0
    _set_fanouts(m, 5)
    monkeypatch.setattr(torch.cuda, "is_current_stream_capturing", lambda: True)
    with pytest.raises(NotImplementedError, match="CUDA graph"):
        m.sampled_minibatch_train_step(indptr, indices, ids, labels)
    with pytest.raises(NotImplementedError, match="CUDA graph"):
        m.sampled_minibatch_embeddings(indptr, indices, ids)
    assert sampler.counter == 0
