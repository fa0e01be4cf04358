"""GPU: full-batch training over whole neighbourhoods.  gs_csr_transpose, GS_CSR_SUM and both phases of
gs_csr_max_backward bit for bit against oracle/full_neighbor_grad.py; SupervisedGraphsage.full_neighbor_outputs equal to
full_neighbor_embeddings; loss and every gradient against the oracle's backward (itself checked against float64 autograd
on the CPU); Adam steps, agreement with the sampled loss where sampling draws whole rows, determinism, the refusals, a
memory bound and a toy-ppi run."""
import numpy as np
import pytest
import torch

from conftest import load_golden, rel_err
from oracle import full_neighbor as fn
from oracle import full_neighbor_grad as fg
from oracle import numerics as nu
from test_zz_gpu_full_neighbor import dev, edge_csr, oracle_aggs

pytestmark = pytest.mark.gpu
GRAD_TOL = 2e-4


@pytest.fixture(scope="module")
def gs():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    import graphsage_b200
    graphsage_b200._lib.lib()
    return graphsage_b200


def hub_csr(rs, n, hub_in=0):
    """edge_csr's rows (degrees 0 .. 600, duplicates, self loops, out-of-range entries) plus, with hub_in, hub_in entries
    pointing at node 3 spread over the other rows (an in-degree hub)."""
    indptr, indices = edge_csr(rs, n, n)
    if not hub_in:
        return indptr, indices
    rows = [list(indices[indptr[i]:indptr[i + 1]]) for i in range(n)]
    for k in range(hub_in):
        rows[(k * 7919) % n].append(3)
    indptr = np.concatenate([[0], np.cumsum([len(r) for r in rows])]).astype(np.int64)
    return indptr, np.array([x for r in rows for x in r], dtype=np.int32)


# ---------------------------------------------------------------- kernels, bit for bit
@pytest.mark.parametrize("with_self", [False, True])
@pytest.mark.parametrize("case", ["messy", "empty", "hub"])
def test_transpose_bit_exact(gs, with_self, case):
    rs = np.random.RandomState(1)
    if case == "empty":
        indptr, indices = np.zeros(51, np.int64), np.zeros(0, np.int32)
    else:
        indptr, indices = hub_csr(rs, 2000, 100000 if case == "hub" else 0)
    t_indptr, t_indices = gs.ops.csr_transpose(dev(indptr), dev(indices), with_self=with_self)
    want_ptr, want_idx = fg.csr_transpose(indptr, indices, with_self)
    assert np.array_equal(t_indptr.cpu().numpy(), want_ptr)
    assert np.array_equal(t_indices[:int(want_ptr[-1])].cpu().numpy(), want_idx)
    if case == "hub":
        assert want_ptr[4] - want_ptr[3] >= 100000
    again = gs.ops.csr_transpose(dev(indptr), dev(indices), with_self=with_self)
    assert torch.equal(again[0], t_indptr) and torch.equal(again[1], t_indices)


@pytest.mark.parametrize("odd", [False, True])
@pytest.mark.parametrize("F", [1, 5, 256, 602])
def test_csr_sum_bit_exact(gs, F, odd):
    rs = np.random.RandomState(F)
    n = 1500
    indptr, indices = hub_csr(rs, n, 20000)
    indices[indices == 11] = 12                                          # node 11 is nobody's neighbour: an empty row
    t_indptr, t_indices = fg.csr_transpose(indptr, indices)           # empty, short and hub rows (in-degree 2 * 10^4)
    x = rs.randn(n + 1, F).astype(np.float32)
    pitch = F + 1 if odd and F % 2 == 0 else F + 2 if odd else (F + 7) // 8 * 8
    t = torch.full((n + 1, pitch), 7.0, device="cuda")
    t[:, :F] = dev(x)
    got = gs.ops.csr_aggregate(t[:, :F], dev(t_indptr), dev(t_indices.astype(np.int32)), "sum")
    want = fg.csr_sum(x, t_indptr, t_indices)
    assert nu.bits_equal(got.cpu().numpy(), want)
    assert np.count_nonzero(np.diff(t_indptr) == 0) > 0                # rows with no entries: +0
    with pytest.raises(ValueError, match="float32"):
        gs.ops.csr_aggregate(t[:, :F].to(torch.bfloat16) if F % 8 == 0 else t[:, :F].half(), dev(t_indptr),
                             dev(t_indices.astype(np.int32)), "sum")


@pytest.mark.parametrize("F", [5, 96, 512])
def test_max_backward_bit_exact_on_ties(gs, F):
    rs = np.random.RandomState(F + 1)
    n = 1200
    indptr, indices = hub_csr(rs, n, 5000)
    z = rs.randint(0, 4, size=(n + 1, F)).astype(np.float32)          # four values: ties everywhere, zeros masked
    m = fn.csr_aggregate(z, indptr, indices, "max")
    dm = rs.randn(n + 1, F).astype(np.float32)
    want_s, want_dz = fg.max_backward(z, m, dm, indptr, indices)
    t_indptr, t_indices = gs.ops.csr_transpose(dev(indptr), dev(indices))
    s = torch.empty((n + 1, F + 3), device="cuda")
    got = gs.ops.csr_max_backward(dev(z), dev(m), dev(dm), dev(indptr), dev(indices), t_indptr, t_indices, s=s)
    assert nu.bits_equal(s[:, :F].cpu().numpy(), want_s)
    assert nu.bits_equal(got.cpu().numpy(), want_dz)


# ---------------------------------------------------------------- the model
def sup_model(gs, kind, concat=True, math="fp32", table="fp32", identity_dim=0, layers=2, n=300, F=20, seed=0, adj=None,
              fanout=5, C=4, weight_decay=0.01, sigmoid=False):
    rs = np.random.RandomState(seed)
    feats = np.vstack([rs.randn(n, F).astype(np.float32), np.zeros((1, F), np.float32)])
    gs.set_default_math(math)
    gs.inits.manual_seed(seed + 1)
    if adj is None:
        adj = rs.randint(0, n, size=(n + 1, 8)).astype(np.int32)
        adj[n] = n
    adj = dev(adj)
    sampler = gs.UniformNeighborSampler(adj, seed=3)
    infos = [gs.SAGEInfo("node", sampler, fanout, d) for d in [16, 12, 8][:layers]]
    f = dev(feats) if table == "fp32" else dev(feats).to(torch.bfloat16)
    m = gs.SupervisedGraphsage(C, {"batch_size": 8, "dropout": 0.}, f, adj, None, infos, concat=concat,
                               aggregator_type=kind, identity_dim=identity_dim, weight_decay=weight_decay,
                               sigmoid_loss=sigmoid)
    gs.set_default_math("fp32")
    return m


def oracle_step(m, indptr, indices, ids, labels):
    feats = m.features.float().cpu().numpy()
    return fg.full_neighbor_loss_grads(feats, indptr, indices, oracle_aggs(m), m.concat, ids, labels,
                                       m.node_pred_vars["weights"].detach().cpu().numpy(),
                                       m.node_pred_vars["bias"].detach().cpu().numpy(), m.sigmoid_loss, m.weight_decay,
                                       m.identity_dim)


def named_grads(m):
    out = []
    for l, a in enumerate(m.aggregators):
        for k, v in a.vars.items():
            out.append(((l, k), v))
        if hasattr(a, "mlp_layers"):
            out += [((l, "mlp_weights"), a.mlp_layers[0].vars["weights"]), ((l, "mlp_bias"), a.mlp_layers[0].vars["bias"])]
    return out + [(("head", "weights"), m.node_pred_vars["weights"]), (("head", "bias"), m.node_pred_vars["bias"])]


# The pools' dbm is a column sum over every node of terms that sit on a ReLU (and for max-pool a tie) discontinuity: one
# pre-activation whose rounding differs from numpy's across zero moves a whole term, which dWm (weighted by the input rows)
# barely shows but the plain sum does.  Its bound is relative to its largest element like the rest, only looser.
POOL_BIAS_TOL = 5e-3


def check_grads(m, grads, head, demb):
    for (l, k), v in named_grads(m):
        ref = head[k] if l == "head" else grads[l][k]
        assert v.grad is not None, (l, k)
        tol = POOL_BIAS_TOL if k == "mlp_bias" else GRAD_TOL
        assert rel_err(v.grad.cpu().numpy(), ref) < tol, (l, k, rel_err(v.grad.cpu().numpy(), ref))
    if demb is not None:
        assert rel_err(m.embeds.grad.cpu().numpy(), demb) < GRAD_TOL


MODEL_CASES = ([(k, c, "fp32", "fp32", 0, 2) for k in ("mean", "maxpool", "meanpool") for c in (False, True)]
               + [("gcn", False, "fp32", "fp32", 0, 2), ("mean", True, "tf32x3", "fp32", 0, 2),
                  ("maxpool", True, "tf32x3", "fp32", 0, 2), ("gcn", False, "tf32x3", "fp32", 0, 2),
                  ("mean", True, "fp32", "bf16", 0, 2), ("maxpool", False, "fp32", "bf16", 0, 2),
                  ("gcn", False, "fp32", "bf16", 0, 2), ("meanpool", True, "fp32", "bf16", 0, 2),
                  ("mean", True, "fp32", "fp32", 16, 2), ("maxpool", True, "fp32", "fp32", 16, 2),
                  ("gcn", False, "tf32x3", "fp32", 16, 2), ("meanpool", False, "fp32", "fp32", 16, 2),
                  ("mean", True, "fp32", "fp32", 0, 3), ("maxpool", True, "tf32x3", "fp32", 0, 3),
                  ("gcn", False, "fp32", "fp32", 16, 3)])


@pytest.mark.parametrize("kind,concat,math,table,identity_dim,layers", MODEL_CASES)
def test_loss_and_gradients_match_the_oracle(gs, kind, concat, math, table, identity_dim, layers):
    m = sup_model(gs, kind, concat, math, table, identity_dim, layers, sigmoid=layers == 3)
    indptr, indices = edge_csr(np.random.RandomState(1), 300, 300)
    ids = np.array([0, 5, 299, 17, 17, 4, 150, 6, 1, 2, 3], dtype=np.int32)
    labels = np.eye(4, dtype=np.float32)[np.arange(len(ids)) % 4]
    out = m.full_neighbor_outputs(dev(indptr), dev(indices), ids)
    assert torch.equal(out.detach(), m.full_neighbor_embeddings(dev(indptr), dev(indices), ids))
    loss = m.full_neighbor_loss(dev(indptr), dev(indices), ids, labels)
    loss.backward()
    rl, grads, head, demb = oracle_step(m, indptr, indices, ids, labels)
    assert abs(float(loss.detach()) - rl) < GRAD_TOL * max(1.0, abs(rl))
    check_grads(m, grads, head, demb)


@pytest.mark.parametrize("kind", ["mean", "maxpool"])
def test_five_adam_steps_track_the_cpu_run(gs, kind):
    m = sup_model(gs, kind, identity_dim=8)
    indptr, indices = edge_csr(np.random.RandomState(2), 300, 300)
    ids = np.arange(0, 300, 3, dtype=np.int32)
    labels = np.eye(4, dtype=np.float32)[ids % 4]
    cpu = [p.detach().cpu().clone().requires_grad_(True) for p in m.parameters()]
    opt = torch.optim.Adam(cpu, lr=m.learning_rate)
    d_indptr, d_indices = dev(indptr), dev(indices)
    for _ in range(5):
        # the CPU run: the oracle's gradients at the CPU parameters, clipped, then torch's Adam on the CPU
        for p, c in zip(m.parameters(), cpu):
            with torch.no_grad():
                p.copy_(c.detach().to(p.device))
        rl, grads, head, demb = oracle_step(m, indptr, indices, ids, labels)
        refs = {id(v): (head[k] if l == "head" else grads[l][k]) for (l, k), v in named_grads(m)}
        if demb is not None:
            refs[id(m.embeds)] = demb
        for p, c in zip(m.parameters(), cpu):
            c.grad = torch.from_numpy(np.asarray(refs[id(p)], np.float32)).clamp(-5.0, 5.0)
        opt.step()
    # the GPU run from the same start
    m2 = sup_model(gs, kind, identity_dim=8)
    for _ in range(5):
        loss = m2.full_neighbor_train_step(d_indptr, d_indices, ids, labels)
    assert loss.dim() == 0 and loss.is_cuda
    for p, c in zip(m2.parameters(), cpu):      # Adam's normalised step amplifies differences in near-zero gradients
        assert rel_err(p.detach().cpu().numpy(), c.detach().numpy()) < 1e-2


@pytest.mark.parametrize("kind", ["mean", "gcn", "maxpool", "meanpool"])
def test_regular_graph_matches_the_sampled_loss(gs, kind):
    n, d = 200, 6
    rs = np.random.RandomState(4)
    indices = np.concatenate([rs.choice(n, d, replace=False) for _ in range(n)]).astype(np.int32)
    indptr = np.arange(n + 1, dtype=np.int64) * d
    adj = np.full((n + 1, d), n, dtype=np.int32)
    for v in range(n):
        adj[v] = rs.permutation(indices[v * d:(v + 1) * d])
    m = sup_model(gs, kind, concat=kind != "gcn", n=n, adj=adj, fanout=d)
    ids = np.arange(0, n, 2, dtype=np.int32)
    labels = np.eye(4, dtype=np.float32)[ids % 4]
    full = m.full_neighbor_loss(indptr, indices, ids, labels)
    full.backward()
    g_full = [p.grad.clone() for p in m.parameters()]
    m.optimizer.zero_grad(set_to_none=True)
    sampled = m.loss(torch.from_numpy(ids), torch.from_numpy(labels))
    sampled.backward()
    assert abs(float(full.detach()) - float(sampled.detach())) < 1e-4 * max(1.0, abs(float(sampled.detach())))
    for a, p in zip(g_full, m.parameters()):
        assert rel_err(a.cpu().numpy(), p.grad.cpu().numpy()) < 1e-3


@pytest.mark.parametrize("kind", ["mean", "maxpool"])
def test_two_steps_from_the_same_state_are_bit_identical(gs, kind):
    indptr, indices = (dev(a) for a in edge_csr(np.random.RandomState(3), 300, 300))
    ids = np.arange(0, 300, 2, dtype=np.int32)
    labels = np.eye(4, dtype=np.float32)[ids % 4]
    runs = []
    for _ in range(2):
        m = sup_model(gs, kind, identity_dim=8)
        losses = [m.full_neighbor_train_step(indptr, indices, ids, labels) for _ in range(2)]
        runs.append((losses, [p.detach().clone() for p in m.parameters()]))
    assert all(torch.equal(a, b) for a, b in zip(runs[0][0], runs[1][0]))
    assert all(torch.equal(a, b) for a, b in zip(runs[0][1], runs[1][1]))


def test_refusals(gs, monkeypatch):
    indptr, indices = edge_csr(np.random.RandomState(0), 300, 300)
    ids, labels = np.arange(4, dtype=np.int32), np.eye(4, dtype=np.float32)
    m = sup_model(gs, "mean")
    m.dropout_rate = 0.5
    with pytest.raises(NotImplementedError, match="dropout"):
        m.full_neighbor_train_step(indptr, indices, ids, labels)
    m.dropout_rate = 0.
    with pytest.raises(ValueError, match="N \\+ 1"):
        m.full_neighbor_loss(indptr[:-1], indices, ids, labels)
    with pytest.raises(TypeError, match="indices"):
        m.full_neighbor_loss(indptr, indices.astype(np.int64), ids, labels)
    monkeypatch.setattr(torch.cuda, "is_current_stream_capturing", lambda: True)
    with pytest.raises(NotImplementedError, match="CUDA graph"):
        m.full_neighbor_train_step(indptr, indices, ids, labels)


def test_peak_memory_bound(gs):
    n, F = 20000, 128
    rs = np.random.RandomState(5)
    deg = rs.randint(1, 60, size=n)
    indptr = np.concatenate([[0], np.cumsum(deg)]).astype(np.int64)
    indices = rs.randint(0, n, size=int(indptr[-1])).astype(np.int32)
    m = sup_model(gs, "maxpool", n=n, F=F, adj=np.full((n + 1, 8), n, np.int32))
    ids = np.arange(n, dtype=np.int32)
    labels = np.eye(4, dtype=np.float32)[ids % 4]
    d_indptr, d_indices = dev(indptr), dev(indices)
    m.full_neighbor_train_step(d_indptr, d_indices, ids, labels)             # transposes built, Adam state allocated
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    m.full_neighbor_train_step(d_indptr, d_indices, ids, labels)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    # per node: the [N+1, 512] MLP outputs, maxes and their gradients of both layers, at most 12 fp32 rows of 512
    bound = (n + 1) * 4 * (12 * 512 + 8 * F + 64)      # a per-entry [E, 512] buffer would be twice this
    assert peak < bound, (peak, bound)


def test_toy_ppi_full_batch_training(gs):
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
    m = gs.SupervisedGraphsage(labels.shape[1], {"batch_size": 64, "dropout": 0.}, feats, dev(it.adj), None, infos,
                               aggregator_type="mean", sigmoid_loss=True, learning_rate=0.01)
    train = np.array([id2idx[u] for u in G.nodes() if not G.node[u]["val"] and not G.node[u]["test"]], dtype=np.int32)
    val = np.array([id2idx[u] for u in G.nodes() if G.node[u]["val"]], dtype=np.int32)
    tr_ptr, tr_idx = it.neighbor_csr(test=False)
    te_ptr, te_idx = it.neighbor_csr(test=True)
    before = calc_f1(labels[val], m.full_neighbor_predict(te_ptr, te_idx, val).cpu().numpy(), True)[0]
    d_ptr, d_idx, d_lab = dev(tr_ptr), dev(tr_idx), dev(labels[train])
    losses = [float(m.full_neighbor_train_step(d_ptr, d_idx, train, d_lab)) for _ in range(20)]
    after = calc_f1(labels[val], m.full_neighbor_predict(te_ptr, te_idx, val).cpu().numpy(), True)[0]
    print("toy-ppi full-batch: loss %.4f -> %.4f, val F1 micro %.4f -> %.4f" % (losses[0], losses[-1], before, after))
    assert losses[-1] < losses[0]
    assert after > before
