"""GPU: full-neighbourhood training with dropout.  gs_csr_aggregate_dropout (mean, mean_self, the transposed sum),
gs_csr_transpose's t_slot and the positioned gs_dropout_apply bit for bit against oracle/full_neighbor_dropout.py; the
model's loss and gradients against the masked oracle; minibatch rows equal to the whole-graph rows; dropout=0 equal to
dropout=None; determinism, the kept fraction, no host synchronisation and a memory bound."""
import numpy as np
import pytest
import torch

from conftest import rel_err
from oracle import full_neighbor_dropout as fd
from oracle.dropout import apply as drop_rows
from test_zz_gpu_full_neighbor import dev, edge_csr, oracle_aggs
from test_zz_gpu_full_neighbor_train import GRAD_TOL, check_grads, sup_model

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def gs():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    import graphsage_b200
    graphsage_b200._lib.lib()
    return graphsage_b200


def degree_csr(rs, n, degrees):
    """Rows of the given degrees (cycled), entries in [-2, n + 3): out-of-range entries, duplicates, self loops."""
    rows = [list(rs.randint(-2, n + 3, size=degrees[i % len(degrees)])) for i in range(n)]
    indptr = np.concatenate([[0], np.cumsum([len(r) for r in rows])]).astype(np.int64)
    return indptr, np.array([x for r in rows for x in r], dtype=np.int32)


DEGREES = [0, 1, 31, 32, 33, 257, 600]


def table(rs, n_rows, F, dtype, odd):
    x = rs.randn(n_rows, F).astype(np.float32)
    if dtype == "bf16":
        t = torch.zeros((n_rows, (F + 7) // 8 * 8), dtype=torch.bfloat16, device="cuda")
        t[:, :F] = dev(x).to(torch.bfloat16)
        return t[:, :F], t[:, :F].float().cpu().numpy()
    pitch = F + 1 if odd else (F + 3) // 4 * 4
    t = torch.zeros((n_rows, pitch), device="cuda")
    t[:, :F] = dev(x)
    return t[:, :F], x


@pytest.mark.parametrize("op", ["mean", "mean_self"])
@pytest.mark.parametrize("dtype,odd", [("fp32", False), ("fp32", True), ("bf16", False)])
@pytest.mark.parametrize("F", [1, 5, 602])
@pytest.mark.parametrize("p", [0.1, 0.5, 0.9])
def test_masked_aggregate_bit_exact(gs, op, dtype, odd, F, p):
    if dtype == "bf16" and F != 602 and p != 0.5:
        pytest.skip("bf16 needs 8-column rows: F = 602 covers it, the narrow widths at p = 0.5")
    rs = np.random.RandomState(F)
    n = 60
    indptr, indices = degree_csr(rs, n, DEGREES)
    src, x = table(rs, n + 1, F, dtype, odd)
    neigh, selfs = (9, 3, p), (9, 4, p)
    pm = (dev(indptr), None, len(indices))
    got = gs.ops.csr_aggregate(src, dev(indptr), dev(indices), op, dropout=(neigh, selfs, pm))
    want = fd.csr_aggregate_dropout(x, indptr, indices, op, neigh, selfs, (indptr, None, len(indices)))
    assert np.array_equal(got.cpu().numpy(), want)
    # rows and a position map: a local CSR whose rows are named through pos_ids
    rows = np.array([3, 0, 59, 60, 5, 5, -1, 44], np.int32)
    pos_ids = rs.permutation(n + 1).astype(np.int32)
    got = gs.ops.csr_aggregate(src, dev(indptr), dev(indices), op, rows=dev(rows),
                               dropout=(neigh, selfs, (dev(indptr * 3), dev(pos_ids), 12345)))
    want = fd.csr_aggregate_dropout(x, indptr, indices, op, neigh, selfs, (indptr * 3, pos_ids, 12345), rows)
    assert np.array_equal(got.cpu().numpy(), want)


def test_hub_row_and_rate_zero(gs):
    rs = np.random.RandomState(2)
    n, F = 40, 37
    rows = [list(rs.randint(0, n, size=100000 if i == 7 else 3)) for i in range(n)]
    indptr = np.concatenate([[0], np.cumsum([len(r) for r in rows])]).astype(np.int64)
    indices = np.array([x for r in rows for x in r], dtype=np.int32)
    src, x = table(rs, n + 1, F, "fp32", False)
    pm = (dev(indptr), None, len(indices))
    for op in ("mean", "mean_self"):
        got = gs.ops.csr_aggregate(src, dev(indptr), dev(indices), op, dropout=((1, 2, 0.5), (1, 3, 0.5), pm))
        want = fd.csr_aggregate_dropout(x, indptr, indices, op, (1, 2, 0.5), (1, 3, 0.5), (indptr, None, len(indices)))
        assert np.array_equal(got.cpu().numpy(), want), op
        zero = gs.ops.csr_aggregate(src, dev(indptr), dev(indices), op, dropout=((1, 2, 0.), (1, 3, 0.), pm))
        assert torch.equal(zero, gs.ops.csr_aggregate(src, dev(indptr), dev(indices), op))


@pytest.mark.parametrize("with_self", [False, True])
def test_transpose_slots_and_masked_sum(gs, with_self):
    rs = np.random.RandomState(3)
    n = 500
    indptr, indices = degree_csr(rs, n, DEGREES)
    t_indptr, t_indices, t_slot = gs.ops.csr_transpose(dev(indptr), dev(indices), with_self=with_self, slots=True)
    plain = gs.ops.csr_transpose(dev(indptr), dev(indices), with_self=with_self)
    assert torch.equal(plain[0], t_indptr) and torch.equal(plain[1], t_indices)         # the same bytes, tail included
    wp, wi, ws = fd.csr_transpose_slots(indptr, indices, with_self)
    E = int(wp[-1])
    assert np.array_equal(t_indptr.cpu().numpy(), wp) and np.array_equal(t_indices[:E].cpu().numpy(), wi)
    assert np.array_equal(t_slot[:E].cpu().numpy(), ws)
    for F, odd in ((5, True), (128, False)):
        g = torch.zeros((n + 1, F + (1 if odd else 0)), device="cuda")
        g[:, :F] = torch.randn((n + 1, F), device="cuda")
        g = g[:, :F]
        pm = (dev(indptr), None, len(indices))
        got = gs.ops.csr_aggregate(g, t_indptr, t_indices, "sum", dropout=((4, 5, 0.5), (4, 6, 0.3), pm), t_slot=t_slot)
        want = fd.csr_sum_dropout(g.cpu().numpy(), wp, wi, ws, (4, 5, 0.5), (4, 6, 0.3), (indptr, None, len(indices)))
        assert np.array_equal(got.cpu().numpy(), want)


def test_positioned_dropout_apply(gs):
    x = torch.randn((300, 37), device="cuda")
    ids = torch.randint(0, 10**6, (300,), dtype=torch.int32, device="cuda")
    got = gs.ops.dropout_apply(x, (3, 8, 0.4), pos_ids=ids)
    want = drop_rows(x.cpu().numpy(), 3, 8, 0.4, pos=ids.cpu().numpy())
    assert np.array_equal(got.cpu().numpy(), want)
    assert torch.equal(gs.ops.dropout_apply(x, (3, 8, 0.4), pos_ids=torch.arange(300, dtype=torch.int32, device="cuda")),
                       gs.ops.dropout_apply(x, (3, 8, 0.4)))


MODEL_CASES = ([(k, c, "fp32", "fp32", 0, 2) for k in ("mean", "maxpool", "meanpool") for c in (False, True)]
               + [("gcn", False, "fp32", "fp32", 0, 2)]
               + [("mean", True, "tf32x3", "fp32", 16, 2), ("maxpool", True, "tf32x3", "fp32", 0, 3),
                  ("gcn", False, "fp32", "bf16", 0, 2), ("meanpool", True, "fp32", "bf16", 0, 2),
                  ("mean", False, "fp32", "bf16", 0, 1), ("gcn", False, "tf32x3", "fp32", 16, 3),
                  ("maxpool", False, "fp32", "fp32", 16, 1), ("meanpool", False, "tf32x3", "fp32", 0, 3)])


@pytest.mark.parametrize("kind,concat,math,table_dtype,identity_dim,layers", MODEL_CASES)
def test_loss_and_gradients_match_the_masked_oracle(gs, kind, concat, math, table_dtype, identity_dim, layers):
    m = sup_model(gs, kind, concat, math, table_dtype, identity_dim, layers)
    indptr, indices = edge_csr(np.random.RandomState(1), 300, 300)
    ids = np.array([0, 5, 299, 17, 17, 4, 150, 6, 1, 2, 3], dtype=np.int32)
    labels = np.eye(4, dtype=np.float32)[np.arange(len(ids)) % 4]
    m.dropout_counter = 21
    loss = m.full_neighbor_loss(dev(indptr), dev(indices), ids, labels, dropout=0.5)
    loss.backward()
    sites = fd.sites(kind, layers, True, m.dropout_key, 21, 0.5)
    feats = m.features.float().cpu().numpy()
    rl, grads, head, demb = fd.full_neighbor_loss_grads(
        feats, indptr, indices, oracle_aggs(m), m.concat, ids, labels, m.node_pred_vars["weights"].detach().cpu().numpy(),
        m.node_pred_vars["bias"].detach().cpu().numpy(), sites, m.sigmoid_loss, m.weight_decay, m.identity_dim)
    assert abs(float(loss.detach()) - rl) < GRAD_TOL * max(1.0, abs(rl))
    check_grads(m, grads, head, demb)


@pytest.mark.parametrize("kind", ["mean", "gcn", "maxpool", "meanpool"])
@pytest.mark.parametrize("layers", [1, 2, 3])
def test_minibatch_equals_the_whole_graph(gs, kind, layers):
    m = sup_model(gs, kind, kind != "gcn", "tf32x3", identity_dim=16 if layers == 2 else 0, layers=layers)
    indptr, indices = edge_csr(np.random.RandomState(2), 300, 300)
    ids = np.array([7, 0, 299, 17, 17, 150, -3, 400], dtype=np.int32)
    m.dropout_counter = 4
    whole = m.full_neighbor_outputs(dev(indptr), dev(indices), ids, dropout=0.3)
    whole.sum().backward()
    gw = [p.grad.clone() for p in m.parameters() if p.grad is not None]
    m.optimizer.zero_grad(set_to_none=True)
    m.dropout_counter = 4
    mini = m.full_neighbor_minibatch_outputs(dev(indptr), dev(indices), ids, dropout=0.3)
    assert torch.equal(whole, mini)
    mini.sum().backward()
    gm = [p.grad.clone() for p in m.parameters() if p.grad is not None]
    for a, b in zip(gw, gm):
        assert rel_err(b.cpu().numpy(), a.cpu().numpy()) < GRAD_TOL


def test_unsupervised_minibatch_loss_equals_the_whole_graph_loss(gs):
    rs = np.random.RandomState(5)
    n, F = 300, 20
    feats = np.vstack([rs.randn(n, F).astype(np.float32), np.zeros((1, F), np.float32)])
    adj = dev(np.vstack([rs.randint(0, n, size=(n, 8)), np.full((1, 8), n)]).astype(np.int32))
    sampler = gs.UniformNeighborSampler(adj, seed=3)
    infos = [gs.SAGEInfo("node", sampler, 5, 16), gs.SAGEInfo("node", sampler, 5, 8)]
    m = gs.UnsupervisedGraphsage({"batch_size": 8, "dropout": 0.5}, dev(feats), adj, np.ones(n), infos,
                                 aggregator_type="mean", neg_sample_size=6)
    indptr, indices = edge_csr(np.random.RandomState(6), n, n)
    b1, b2 = np.array([1, 2, 3, 4], np.int32), np.array([5, 6, 7, 299], np.int32)
    c0, s0 = m.dropout_counter, m.neg_sampler.counter
    loss = m.full_neighbor_minibatch_loss(dev(indptr), dev(indices), b1, b2, dropout=m.dropout_rate)
    m.neg_sampler.counter, m.dropout_counter = s0, c0
    neg = m.neg_sampler(m.neg_sample_size)
    from graphsage_b200.full_neighbor_training import full_neighbor_outputs
    out = full_neighbor_outputs(m, dev(indptr), dev(indices), torch.cat([dev(b1), dev(b2), neg]), dropout=0.5)
    ref = m._pairs_loss(*torch.split(out, [4, 4, neg.numel()]))
    assert torch.equal(loss, ref)


def test_rate_zero_determinism_fraction_inference_and_no_sync(gs):
    indptr, indices = edge_csr(np.random.RandomState(7), 300, 300)
    ids = np.arange(0, 300, 3, dtype=np.int32)
    labels = np.eye(4, dtype=np.float32)[np.arange(len(ids)) % 4]
    a, b = sup_model(gs, "mean"), sup_model(gs, "mean")
    assert torch.equal(a.full_neighbor_outputs(dev(indptr), dev(indices), ids, dropout=0.),
                       a.full_neighbor_outputs(dev(indptr), dev(indices), ids))
    losses = []
    for m in (a, b):
        losses.append([float(m.full_neighbor_train_step(dev(indptr), dev(indices), ids, labels, dropout=0.5))
                       for _ in range(3)])
    assert losses[0] == losses[1]
    for p, q in zip(a.parameters(), b.parameters()):
        assert torch.equal(p, q)
    # inference never drops: a rate > 0 model embeds as its rate-0 twin
    with torch.no_grad():
        b.dropout_rate = 0.5
    assert torch.equal(b.full_neighbor_embeddings(dev(indptr), dev(indices), ids),
                       a.full_neighbor_embeddings(dev(indptr), dev(indices), ids))
    # the kept fraction over >= 10^6 elements
    ones = torch.ones((5000, 256), device="cuda")
    n_rows = ones.shape[0]
    ip = torch.arange(n_rows, dtype=torch.int64, device="cuda")
    ix = torch.arange(n_rows - 1, dtype=torch.int32, device="cuda")
    y = gs.ops.csr_aggregate(ones, ip, ix, "mean", dropout=((3, 1, 0.3), (3, 2, 0.3), (ip, None, n_rows - 1)))
    kept = float((y[:-1] != 0).float().mean())
    assert abs(kept - 0.7) < 5e-3
    ip, ix, ids_d, lab_d = dev(indptr), dev(indices), dev(ids), dev(labels)       # inputs on the device first
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        a.full_neighbor_train_step(ip, ix, ids_d, lab_d, dropout=0.5)
    finally:
        torch.cuda.set_sync_debug_mode("default")


def test_peak_memory_bound(gs):
    n, F = 20000, 64
    rs = np.random.RandomState(8)
    indptr, indices = degree_csr(rs, n, [3, 10, 30])
    ids = np.arange(0, n, 2, dtype=np.int32)
    labels = np.eye(4, dtype=np.float32)[np.arange(len(ids)) % 4]
    peaks = {}
    for p in (0., 0.5):
        m = sup_model(gs, "mean", n=n, F=F)
        ip, ix = dev(indptr), dev(indices)
        m.full_neighbor_train_step(ip, ix, ids, labels, dropout=p)             # caches the transposes
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        m.full_neighbor_train_step(ip, ix, ids, labels, dropout=p)
        torch.cuda.synchronize()
        peaks[p] = torch.cuda.max_memory_allocated() - base
    # one fp32 [N+1, F] copy per masked self input (layer 0: F, layer 1: 2 x 16 concat)
    allowance = (n + 1) * (F + 32) * 4
    assert peaks[0.5] <= peaks[0.] + allowance, (peaks, allowance)
