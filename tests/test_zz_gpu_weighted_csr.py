"""GPU: aggregation over weighted edges.  gs_csr_aggregate_weighted (every op, fp32 and bf16 sources), the weighted
transposed sum and gs_csr_max_backward_weighted bit for bit against oracle/weighted.py; all-one weights torch.equal to the
unweighted kernels; the models' embeddings against the oracle, minibatch and sampled rows torch.equal to the whole
graph's, losses and gradients against the oracle's backward (itself checked against float64 autograd on the CPU), Adam
steps, determinism, a whole-graph step free of host synchronisation, and the refusals."""
import numpy as np
import pytest
import torch

from conftest import rel_err
from oracle import full_neighbor_grad as fg
from oracle import numerics as nu
from oracle import pool2_forward as p2
from oracle import weighted as ow
from test_zz_gpu_full_neighbor import dev, edge_csr, oracle_aggs, table_of
from test_zz_gpu_full_neighbor_train import GRAD_TOL, POOL_BIAS_TOL, hub_csr, named_grads, sup_model
from test_zz_gpu_sampled_blocks import _set_fanouts

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def gs():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    import graphsage_b200
    graphsage_b200._lib.lib()
    return graphsage_b200


def weights_of(rs, n, kind):
    if kind == "one":
        return np.ones(n, np.float32)
    if kind == "zero":
        return np.zeros(n, np.float32)
    if kind == "negative":
        return -(rs.rand(n) * 3).astype(np.float32)
    w = (rs.randn(n) * 2).astype(np.float32)
    w[::9] = 0
    return w


WKINDS = ["one", "random", "zero", "negative"]


def same_bits(got, want, op):
    """Bit equality; for the max, +0 and -0 are one value (fmaxf's choice between fl(0 * x) of both signs is
    unspecified, and every reader of m - the GEMM, the tie test of the backward - treats them alike)."""
    if op == "max":
        got, want = got + np.float32(0), want + np.float32(0)
    return nu.bits_equal(got, want)


def capped(indptr, indices, cap=256):
    """The rows cut to their first cap entries (sampled blocks take fanouts up to 256)."""
    deg = np.minimum(np.diff(indptr), cap)
    keep = np.concatenate([np.arange(indptr[v], indptr[v] + deg[v]) for v in range(len(deg))])
    return np.concatenate([[0], np.cumsum(deg)]).astype(np.int64), indices[keep]


# ---------------------------------------------------------------- kernels, bit for bit
@pytest.mark.parametrize("wkind", WKINDS)
@pytest.mark.parametrize("dtype,F", [("fp32", 1), ("fp32", 5), ("fp32", 602), ("fp32", 1024), ("fp32_odd", 5),
                                     ("bf16", 5), ("bf16", 602)])
@pytest.mark.parametrize("op", ["mean", "mean_self", "max"])
def test_weighted_aggregate_bit_exact(gs, op, dtype, F, wkind):
    rs = np.random.RandomState(F + len(wkind))
    n = 1500
    indptr, indices = edge_csr(rs, n, n + 1)              # degrees 0, 1, 31, 32, 33, 257, 600; out-of-range entries
    src, x = table_of(rs, n + 1, F, dtype)
    w = weights_of(rs, len(indices), wkind)
    got = gs.ops.csr_aggregate(src, dev(indptr), dev(indices), op, weights=dev(w))
    want = ow.csr_aggregate(x, indptr, indices, op, None, w)
    assert same_bits(got.cpu().numpy(), want, op)
    rows = np.array([5, 0, 6, -1, n, n + 9, 3, 3, 1], np.int32)            # a rows subset, out-of-range rows
    got_r = gs.ops.csr_aggregate(src, dev(indptr), dev(indices), op, rows=dev(rows), weights=dev(w))
    assert same_bits(got_r.cpu().numpy(), ow.csr_aggregate(x, indptr, indices, op, rows, w), op)
    again = gs.ops.csr_aggregate(src, dev(indptr), dev(indices), op, weights=dev(w))
    assert torch.equal(again, got)
    if wkind == "one":
        assert torch.equal(got, gs.ops.csr_aggregate(src, dev(indptr), dev(indices), op))


@pytest.mark.parametrize("op", ["mean", "max"])
@pytest.mark.parametrize("F", [5, 602])
def test_weighted_hub_row_bit_exact(gs, op, F):
    rs = np.random.RandomState(3)
    n = 300
    deg = rs.randint(0, 5, size=n)
    deg[7] = 100000                                                        # a 10^5-entry hub row
    indptr = np.concatenate([[0], np.cumsum(deg)]).astype(np.int64)
    indices = rs.randint(0, n, size=int(indptr[-1])).astype(np.int32)
    src, x = table_of(rs, n + 1, F, "fp32")
    w = weights_of(rs, len(indices), "random")
    rows = np.array([7, 1, 7, 2], np.int32)
    got = gs.ops.csr_aggregate(src, dev(indptr), dev(indices), op, rows=dev(rows), weights=dev(w))
    assert same_bits(got.cpu().numpy(), ow.csr_aggregate(x, indptr, indices, op, rows, w), op)


def test_weighted_aggregate_of_an_edgeless_graph(gs):
    rs = np.random.RandomState(4)
    src, x = table_of(rs, 51, 7, "fp32")
    indptr, indices = np.zeros(51, np.int64), np.zeros(0, np.int32)
    for op in ("mean", "mean_self", "max"):
        got = gs.ops.csr_aggregate(src, dev(indptr), dev(indices), op, weights=dev(np.zeros(0, np.float32)))
        assert same_bits(got.cpu().numpy(), ow.csr_aggregate(x, indptr, indices, op, None, np.zeros(0, np.float32)), op)


@pytest.mark.parametrize("with_self", [False, True])
@pytest.mark.parametrize("F", [1, 5, 602])
def test_weighted_sum_over_the_transpose_bit_exact(gs, F, with_self):
    rs = np.random.RandomState(F + with_self)
    n = 1500
    indptr, indices = hub_csr(rs, n, 20000)                               # an in-degree hub of 2 * 10^4
    w = weights_of(rs, len(indices), "random")
    t_indptr, t_indices, t_slot = gs.ops.csr_transpose(dev(indptr), dev(indices), with_self=with_self, slots=True)
    tw = gs.ops.csr_transpose_weights(dev(w), dev(indptr), t_indices, t_slot)
    cnt = int(t_indptr[-1])
    want_tw = ow.transpose_weights(indptr, indices, w, with_self)
    assert nu.bits_equal(tw[:cnt].cpu().numpy(), want_tw)
    g = rs.randn(n + 1, F).astype(np.float32)
    got = gs.ops.csr_aggregate(dev(g), t_indptr, t_indices, "sum", weights=tw)
    want_ptr, want_idx = fg.csr_transpose(indptr, indices, with_self)
    assert nu.bits_equal(got.cpu().numpy(), ow.csr_sum(g, want_ptr, want_idx, want_tw))
    ones = torch.ones_like(tw)
    assert torch.equal(gs.ops.csr_aggregate(dev(g), t_indptr, t_indices, "sum", weights=ones),
                       gs.ops.csr_aggregate(dev(g), t_indptr, t_indices, "sum"))


@pytest.mark.parametrize("wkind", WKINDS)
@pytest.mark.parametrize("F", [5, 96])
def test_weighted_max_backward_bit_exact_on_ties(gs, F, wkind):
    rs = np.random.RandomState(F + 7)
    n = 1200
    indptr, indices = hub_csr(rs, n, 5000)
    z = rs.randint(0, 4, size=(n + 1, F)).astype(np.float32)             # ties everywhere, zeros masked
    w = rs.randint(-1, 3, size=len(indices)).astype(np.float32) if wkind == "random" else \
        weights_of(rs, len(indices), wkind)                              # small integers: exact weighted ties
    m = ow.csr_aggregate(z, indptr, indices, "max", None, w)
    dm = rs.randn(n + 1, F).astype(np.float32)
    want_s, want_dz = ow.max_backward(z, m, dm, indptr, indices, w)
    t_indptr, t_indices, t_slot = gs.ops.csr_transpose(dev(indptr), dev(indices), slots=True)
    tw = gs.ops.csr_transpose_weights(dev(w), dev(indptr), t_indices, t_slot)
    s = torch.empty((n + 1, F + 3), device="cuda")
    got = gs.ops.csr_max_backward(dev(z), dev(m), dev(dm), dev(indptr), dev(indices), t_indptr, t_indices, s=s,
                                  weights=dev(w), t_weights=tw)
    assert nu.bits_equal(s[:, :F].cpu().numpy(), want_s)
    assert nu.bits_equal(got.cpu().numpy(), want_dz)
    if wkind == "one":
        plain = gs.ops.csr_max_backward(dev(z), dev(m), dev(dm), dev(indptr), dev(indices), t_indptr, t_indices)
        assert torch.equal(got, plain)


# ---------------------------------------------------------------- the models
MODEL_CASES = ([(k, c, "fp32", "fp32", 0, 2) for k in ("mean", "maxpool", "meanpool") for c in (False, True)]
               + [("gcn", False, "fp32", "fp32", 0, 2), ("mean", True, "tf32x3", "fp32", 0, 2),
                  ("maxpool", True, "tf32x3", "bf16", 0, 2), ("gcn", False, "fp32", "bf16", 0, 2),
                  ("meanpool", True, "fp32", "bf16", 0, 2), ("mean", True, "fp32", "fp32", 16, 2),
                  ("maxpool", False, "fp32", "fp32", 16, 2), ("gcn", False, "tf32x3", "fp32", 16, 1),
                  ("mean", False, "fp32", "fp32", 0, 1), ("mean", True, "fp32", "fp32", 0, 3),
                  ("maxpool", True, "tf32x3", "fp32", 0, 3)])


def _case(gs, kind, concat, math, table, identity_dim, layers, seed=1):
    m = sup_model(gs, kind, concat, math, table, identity_dim, layers, sigmoid=layers == 3)
    rs = np.random.RandomState(seed)
    indptr, indices = capped(*edge_csr(rs, 300, 300))
    w = weights_of(rs, len(indices), "random")
    return m, indptr, indices, w


def _oracle_step(m, indptr, indices, w, ids, labels):
    return ow.loss_grads(m.features.float().cpu().numpy(), indptr, indices, w, oracle_aggs(m), m.concat, ids, labels,
                         m.node_pred_vars["weights"].detach().cpu().numpy(),
                         m.node_pred_vars["bias"].detach().cpu().numpy(), m.sigmoid_loss, m.weight_decay, m.identity_dim)


def _check_grads(m, grads, head, demb):
    for (l, k), v in named_grads(m):
        ref = head[k] if l == "head" else grads[l][k]
        assert v.grad is not None, (l, k)
        tol = POOL_BIAS_TOL if k == "mlp_bias" else GRAD_TOL
        assert rel_err(v.grad.cpu().numpy(), ref) < tol, (l, k, rel_err(v.grad.cpu().numpy(), ref))
    if demb is not None:
        assert rel_err(m.embeds.grad.cpu().numpy(), demb) < GRAD_TOL


IDS = np.array([0, 5, 299, 17, 17, 4, 150, 6, 1, 2, 3], dtype=np.int32)


@pytest.mark.parametrize("kind,concat,math,table,identity_dim,layers", MODEL_CASES)
def test_embeddings_and_minibatches_match(gs, kind, concat, math, table, identity_dim, layers):
    m, indptr, indices, w = _case(gs, kind, concat, math, table, identity_dim, layers)
    d_ip, d_ix, d_w = dev(indptr), dev(indices), dev(w)
    emb = m.full_neighbor_embeddings(d_ip, d_ix, IDS, edge_weight=d_w)
    ref = ow.embeddings(m.features.float().cpu().numpy(), indptr, indices, w, oracle_aggs(m), concat, IDS)
    assert rel_err(emb.cpu().numpy(), ref) < 1e-4
    assert torch.equal(emb, m.full_neighbor_embeddings(indptr, indices, IDS, edge_weight=w))       # numpy in
    assert torch.equal(emb, m.full_neighbor_minibatch_embeddings(d_ip, d_ix, IDS, edge_weight=d_w))
    _set_fanouts(m, int(np.diff(indptr).max()))
    assert torch.equal(emb, m.sampled_minibatch_embeddings(d_ip, d_ix, IDS, edge_weight=d_w))
    assert not torch.equal(emb, m.full_neighbor_embeddings(d_ip, d_ix, IDS))
    out = m.full_neighbor_outputs(d_ip, d_ix, IDS, edge_weight=d_w)
    assert torch.equal(out.detach(), emb)
    assert torch.equal(m.full_neighbor_minibatch_outputs(d_ip, d_ix, IDS, edge_weight=d_w).detach(), emb)


@pytest.mark.parametrize("kind,concat,math,table,identity_dim,layers", MODEL_CASES)
def test_losses_and_gradients_match_the_oracle(gs, kind, concat, math, table, identity_dim, layers):
    m, indptr, indices, w = _case(gs, kind, concat, math, table, identity_dim, layers)
    labels = np.eye(4, dtype=np.float32)[np.arange(len(IDS)) % 4]
    rl, grads, head, demb = _oracle_step(m, indptr, indices, w, IDS, labels)
    for loss_fn in (m.full_neighbor_loss, m.full_neighbor_minibatch_loss, m.sampled_minibatch_loss):
        m.optimizer.zero_grad(set_to_none=True)
        if loss_fn == m.sampled_minibatch_loss:
            _set_fanouts(m, int(np.diff(indptr).max()))
        loss = loss_fn(dev(indptr), dev(indices), IDS, labels, edge_weight=dev(w))
        loss.backward()
        assert abs(float(loss.detach()) - rl) < GRAD_TOL * max(1.0, abs(rl))
        _check_grads(m, grads, head, demb)


def test_sampled_blocks_with_small_fanouts_match_the_oracle(gs):
    m, indptr, indices, w = _case(gs, "mean", True, "fp32", "fp32", 16, 2)
    m.layer_infos = [info._replace(num_samples=k) for info, k in zip(m.layer_infos, (3, 5))]
    labels = np.eye(4, dtype=np.float32)[np.arange(len(IDS)) % 4]
    sampler = m.layer_infos[0].neigh_sampler
    call = int(sampler.counter)
    loss = m.sampled_minibatch_loss(dev(indptr), dev(indices), IDS, labels, edge_weight=dev(w))
    loss.backward()
    rl, grads, head, demb = ow.loss_grads(m.features.float().cpu().numpy(), indptr, indices, w, oracle_aggs(m), m.concat,
                                          IDS, labels, m.node_pred_vars["weights"].detach().cpu().numpy(),
                                          m.node_pred_vars["bias"].detach().cpu().numpy(), m.sigmoid_loss,
                                          m.weight_decay, m.identity_dim, mode="sampled", fanouts=[3, 5],
                                          seed=int(sampler.seed), call=call)
    assert abs(float(loss.detach()) - rl) < GRAD_TOL * max(1.0, abs(rl))
    _check_grads(m, grads, head, demb)


def test_twomaxpool_inference_matches_the_oracle(gs):
    rs = np.random.RandomState(5)
    n, F = 300, 12
    feats = np.vstack([rs.randn(n, F).astype(np.float32), np.zeros((1, F), np.float32)])
    adj = dev(np.full((n + 1, 4), n, np.int32))
    sampler = gs.UniformNeighborSampler(adj, seed=3)
    infos = [gs.SAGEInfo("node", sampler, 4, 8), gs.SAGEInfo("node", sampler, 4, 8)]
    gs.inits.manual_seed(2)
    m = gs.SupervisedGraphsage(4, {"batch_size": 8, "dropout": 0.}, dev(feats), adj, None, infos, concat=True,
                               aggregator_type="twomaxpool")
    indptr, indices = edge_csr(rs, n, n)
    w = weights_of(rs, len(indices), "random")
    emb = m.full_neighbor_embeddings(dev(indptr), dev(indices), IDS, edge_weight=dev(w))
    aggs = []
    for a in m.aggregators:
        l1, l2 = (l.vars for l in a.mlp_layers)
        d = dict(type="twomaxpool", W1=l1["weights"], b1=l1["bias"], W2=l2["weights"], b2=l2["bias"], **a.vars)
        aggs.append({k: (v.detach().cpu().numpy() if torch.is_tensor(v) else v) for k, v in d.items()})
    ref = ow.embeddings(feats, indptr, indices, w, aggs, True, IDS)
    assert rel_err(emb.cpu().numpy(), ref) < 1e-4
    assert torch.equal(emb, m.full_neighbor_minibatch_embeddings(dev(indptr), dev(indices), IDS, edge_weight=dev(w)))
    one = m.full_neighbor_embeddings(dev(indptr), dev(indices), IDS, edge_weight=torch.ones(len(indices), device="cuda"))
    assert torch.equal(one, m.full_neighbor_embeddings(dev(indptr), dev(indices), IDS))
    ws = [{k: v for k, v in a.items() if k != "type"} for a in aggs]
    assert rel_err(p2.full_neighbor_embeddings(feats, indptr, indices, ws, True, node_ids=IDS),
                   ow.embeddings(feats, indptr, indices, np.ones_like(w), aggs, True, IDS)) < 1e-6


@pytest.mark.parametrize("kind", ["mean", "maxpool"])
def test_unsupervised_losses_match_between_blocks(gs, kind):
    rs = np.random.RandomState(6)
    n, F = 300, 20
    feats = np.vstack([rs.randn(n, F).astype(np.float32), np.zeros((1, F), np.float32)])
    adj = dev(rs.randint(0, n, size=(n + 1, 8)).astype(np.int32))
    indptr, indices = capped(*edge_csr(rs, n, n))
    w = dev(weights_of(rs, len(indices), "random"))
    big = int(np.diff(indptr).max())
    grads = []
    for sampled in (False, True):
        sampler = gs.UniformNeighborSampler(adj, seed=3)
        infos = [gs.SAGEInfo("node", sampler, big, 16), gs.SAGEInfo("node", sampler, big, 16)]
        gs.inits.manual_seed(1)
        m = gs.UnsupervisedGraphsage({"batch_size": 8, "dropout": 0.}, dev(feats), adj, np.ones(n), infos,
                                     concat=True, aggregator_type=kind, neg_sample_size=5)
        b1, b2 = np.arange(0, 16, dtype=np.int32), np.arange(16, 32, dtype=np.int32)
        fn_ = m.sampled_minibatch_loss if sampled else m.full_neighbor_minibatch_loss
        loss = fn_(dev(indptr), dev(indices), b1, b2, edge_weight=w)
        loss.backward()
        grads.append((float(loss.detach()), [p.grad.clone() for p in m.parameters() if p.grad is not None]))
    assert grads[0][0] == grads[1][0]
    assert all(torch.equal(a, b) for a, b in zip(grads[0][1], grads[1][1]))


@pytest.mark.parametrize("kind", ["mean", "maxpool"])
def test_five_adam_steps_track_the_cpu_run(gs, kind):
    m = sup_model(gs, kind, identity_dim=8)
    rs = np.random.RandomState(2)
    indptr, indices = edge_csr(rs, 300, 300)
    w = weights_of(rs, len(indices), "random")
    ids = np.arange(0, 300, 3, dtype=np.int32)
    labels = np.eye(4, dtype=np.float32)[ids % 4]
    cpu = [p.detach().cpu().clone().requires_grad_(True) for p in m.parameters()]
    opt = torch.optim.Adam(cpu, lr=m.learning_rate)
    for _ in range(5):
        for p, c in zip(m.parameters(), cpu):
            with torch.no_grad():
                p.copy_(c.detach().to(p.device))
        rl, grads, head, demb = _oracle_step(m, indptr, indices, w, ids, labels)
        refs = {id(v): (head[k] if l == "head" else grads[l][k]) for (l, k), v in named_grads(m)}
        refs[id(m.embeds)] = demb
        for p, c in zip(m.parameters(), cpu):
            c.grad = torch.from_numpy(np.asarray(refs[id(p)], np.float32)).clamp(-5.0, 5.0)
        opt.step()
    m2 = sup_model(gs, kind, identity_dim=8)
    for _ in range(5):
        loss = m2.full_neighbor_train_step(dev(indptr), dev(indices), ids, labels, edge_weight=dev(w))
    assert loss.dim() == 0 and loss.is_cuda
    for p, c in zip(m2.parameters(), cpu):
        assert rel_err(p.detach().cpu().numpy(), c.detach().numpy()) < 1e-2


@pytest.mark.parametrize("kind", ["mean", "gcn", "maxpool", "meanpool"])
def test_repeated_steps_are_bit_identical_and_free_of_host_synchronisation(gs, kind):
    rs = np.random.RandomState(3)
    indptr, indices = (dev(a) for a in edge_csr(rs, 300, 300))
    w = dev(weights_of(rs, indices.numel(), "random"))
    ids = dev(np.arange(0, 300, 2, dtype=np.int32))
    labels = torch.eye(4, device="cuda")[torch.arange(ids.numel(), device="cuda") % 4]
    runs = []
    for _ in range(2):
        m = sup_model(gs, kind, concat=kind != "gcn", identity_dim=8)
        losses = [m.full_neighbor_train_step(indptr, indices, ids, labels, edge_weight=w)]     # builds the transposes
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            losses.append(m.full_neighbor_train_step(indptr, indices, ids, labels, edge_weight=w))
        finally:
            torch.cuda.set_sync_debug_mode("default")
        runs.append((losses, [p.detach().clone() for p in m.parameters()]))
    assert all(torch.equal(a, b) for a, b in zip(runs[0][0], runs[1][0]))
    assert all(torch.equal(a, b) for a, b in zip(runs[0][1], runs[1][1]))


def test_refusals(gs):
    m, indptr, indices, w = _case(gs, "mean", True, "fp32", "fp32", 0, 2)
    labels = np.eye(4, dtype=np.float32)[np.arange(len(IDS)) % 4]
    for call in (lambda: m.full_neighbor_train_step(indptr, indices, IDS, labels, dropout=0.5, edge_weight=w),
                 lambda: m.full_neighbor_minibatch_loss(indptr, indices, IDS, labels, dropout=0.5, edge_weight=w),
                 lambda: m.sampled_minibatch_loss(indptr, indices, IDS, labels, dropout=0.5, edge_weight=w)):
        with pytest.raises(NotImplementedError, match="edge_weight with training dropout"):
            call()
    with pytest.raises(ValueError, match="device"):
        m.full_neighbor_embeddings(indptr, indices, IDS, edge_weight=torch.from_numpy(w))
    with pytest.raises(ValueError, match="one weight per CSR entry"):
        m.full_neighbor_embeddings(indptr, indices, IDS, edge_weight=w[:-1])
    with pytest.raises(TypeError, match="float32"):
        m.full_neighbor_embeddings(indptr, indices, IDS, edge_weight=w.astype(np.float64))
    m.features = gs.Int8Features(m.features.float())
    with pytest.raises(NotImplementedError, match="full-neighbourhood inference"):          # the existing refusal
        m.full_neighbor_embeddings(indptr, indices, IDS, edge_weight=w)
