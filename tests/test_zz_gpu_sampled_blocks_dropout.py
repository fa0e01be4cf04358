"""GPU: training dropout over sampled blocks.  The fill's per-entry offsets byte for byte against
oracle/sampled_blocks_dropout.py (the other block arrays equal the plain fill's), the masked reduction with offsets and
the remapped transposed sum bit for bit, equality with the masked whole-neighbourhood minibatch when every fanout covers
every row, losses and gradients against the CPU oracle, batch independence, determinism, rates, host reads and a toy-ppi
epoch at p = 0.5."""
import warnings

import numpy as np
import pytest
import torch

from conftest import load_golden, rel_err
from oracle import full_neighbor_dropout as fd
from oracle import sampled_blocks_dropout as sbd
from test_zz_gpu_full_neighbor import dev, edge_csr, oracle_aggs  # noqa: F401
from test_zz_gpu_full_neighbor_minibatch import named_grads_unsup, unsup_model
from test_zz_gpu_full_neighbor_train import POOL_BIAS_TOL, named_grads, sup_model
from test_zz_gpu_sampled_blocks import _check_blocks, _set_fanouts, capped_csr, graph

pytestmark = pytest.mark.gpu
GRAD_TOL = 2e-4


@pytest.fixture(scope="module")
def gs():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    import graphsage_b200
    graphsage_b200._lib.lib()
    return graphsage_b200


# ---------------------------------------------------------------- the fill's offsets, byte for byte
@pytest.mark.parametrize("k", [1, 10, 25, 100, 256])
@pytest.mark.parametrize("name", ["toy-ppi", "rmat", "messy", "empty"])
def test_fill_offsets_bit_exact(gs, name, k):
    indptr, indices = graph(name)
    N = len(indptr) - 1
    rs = np.random.RandomState(k)
    seeds = np.concatenate([rs.randint(0, max(N, 1), size=200), [17, 17, -1, N, N + 4]]).astype(np.int32)
    for L in (1, 2, 3):
        fanouts = [k, max(1, k // 2), k][:L]
        for seed, call in ((123, 0), (123, 1), (2**63 + 7, 0), (2**63 + 7, 5)):
            args = (dev(indptr), dev(indices), dev(seeds), L)
            got, offs = gs.ops.csr_blocks(*args, fanouts=fanouts, seed=seed, call=call, entry_offsets=True)
            plain = gs.ops.csr_blocks(*args, fanouts=fanouts, seed=seed, call=call)
            assert all(torch.equal(a, b) for x, y in zip(got, plain) for a, b in zip(x, y))
            want, want_off = sbd.entry_offsets(indptr, indices, seeds, fanouts, seed, call)
            _check_blocks(got, want)
            for o, w in zip(offs, want_off):
                assert o.dtype == torch.int32 and np.array_equal(o.cpu().numpy(), w)


# ---------------------------------------------------------------- the masked reductions, bit for bit
def _block_case(gs, name, k, seed=4):
    indptr, indices = graph(name)
    N = len(indptr) - 1
    seeds = np.random.RandomState(seed).randint(0, N, size=300).astype(np.int32)
    blocks, offs = gs.ops.csr_blocks(dev(indptr), dev(indices), dev(seeds), 1, fanouts=[k], seed=11, call=seed,
                                     entry_offsets=True)
    return indptr, indices, blocks[0], offs[0]


@pytest.mark.parametrize("dtype", ["fp32", "bf16"])
@pytest.mark.parametrize("op", ["mean", "mean_self"])
@pytest.mark.parametrize("p", [0.1, 0.5, 0.9])
def test_masked_reduction_with_offsets_bit_exact(gs, dtype, op, p):
    for name, k, F in (("rmat", 100, 40), ("rmat", 256, 16), ("toy-ppi", 25, 50), ("messy", 3, 9)):
        indptr, indices, b, off = _block_case(gs, name, k)
        if dtype == "bf16":
            F = (F + 7) // 8 * 8
        n = b.src_ids.numel()
        x = torch.randn((n, F), generator=torch.Generator(device="cuda").manual_seed(k), device="cuda")
        if dtype == "bf16":
            x = x.to(torch.bfloat16)
        ns, ss = (7, 3, p), (7, 4, p)
        pmap = (dev(indptr), b.src_ids, len(indices), off)
        got = gs.ops.csr_aggregate(x, b.indptr, b.indices, op, rows=b.rows, dropout=(ns, ss, pmap))
        want = sbd.csr_aggregate_dropout_offsets(x.float().cpu().numpy(), b.indptr.cpu().numpy(),
                                                 b.indices.cpu().numpy(), op, ns, ss,
                                                 (indptr, b.src_ids.cpu().numpy(), len(indices), off.cpu().numpy()),
                                                 b.rows.cpu().numpy())
        assert np.array_equal(got.cpu().numpy(), want), (name, k)
        if k > 64:                                           # rows above the 64-entry round of the hub schedule
            assert int(torch.diff(b.indptr).max()) > 64


def test_offsets_on_a_hub_row_where_hub_ctas_loop(gs):
    """A hand-built offset array on a 10^5-entry row among 70,000 short rows: hub work items outnumber hub CTAs."""
    rs = np.random.RandomState(3)
    n = 70000
    deg = rs.randint(0, 4, size=n)
    deg[[5, 40000]] = [100000, 300]
    b_indptr = np.concatenate([[0], np.cumsum(deg)]).astype(np.int64)
    b_indices = rs.randint(-1, n + 1, size=int(b_indptr[-1])).astype(np.int32)
    off = np.concatenate([(np.arange(d) * 7919) % max(2 * d, 1) for d in deg]).astype(np.int32)
    g_indptr = np.concatenate([[0], np.cumsum(deg * 2)]).astype(np.int64)          # a "raw" CSR twice as long
    x = torch.randn((n + 1, 64), generator=torch.Generator(device="cuda").manual_seed(1), device="cuda")
    ns, ss = (2, 9, 0.4), (2, 10, 0.4)
    rows = np.concatenate([[5, 40000], rs.randint(0, n + 2, size=3000)]).astype(np.int32)
    for r in (None, rows):
        got = gs.ops.csr_aggregate(x, dev(b_indptr), dev(b_indices), "mean", rows=None if r is None else dev(r),
                                   dropout=(ns, ss, (dev(g_indptr), None, int(g_indptr[-1]), dev(off))))
        want = sbd.csr_aggregate_dropout_offsets(x.cpu().numpy(), b_indptr, b_indices, "mean", ns, ss,
                                                 (g_indptr, None, int(g_indptr[-1]), off), r)
        assert np.array_equal(got.cpu().numpy(), want)


@pytest.mark.parametrize("with_self", [False, True])
def test_remapped_transposed_sum_bit_exact(gs, with_self):
    for name, k in (("rmat", 25), ("messy", 2), ("toy-ppi", 10)):
        indptr, indices, b, off = _block_case(gs, name, k, seed=9)
        t_indptr, t_indices, t_slot = gs.ops.csr_transpose(b.indptr, b.indices, with_self=with_self, slots=True)
        mapped = gs.ops.csr_slots_to_offsets(t_slot, t_indices, b.indptr, off)
        w_ptr, w_idx, w_slot = fd.csr_transpose_slots(b.indptr.cpu().numpy(), b.indices.cpu().numpy(), with_self)
        w_slot = sbd.slots_to_offsets(w_slot, w_idx, b.indptr.cpu().numpy(), off.cpu().numpy())
        cnt = int(w_ptr[-1])
        assert np.array_equal(mapped[:cnt].cpu().numpy(), w_slot)
        n = b.src_ids.numel()
        g = torch.randn((n, 24), generator=torch.Generator(device="cuda").manual_seed(2), device="cuda")
        ns, ss = (5, 1, 0.5), (5, 2, 0.5)
        got = gs.ops.csr_aggregate(g, t_indptr, t_indices, "sum", t_slot=mapped,
                                   dropout=(ns, ss, (dev(indptr), b.src_ids, len(indices))))
        want = fd.csr_sum_dropout(g.cpu().numpy(), w_ptr, w_idx, w_slot, ns, ss,
                                  (indptr, b.src_ids.cpu().numpy(), len(indices)))
        assert np.array_equal(got.cpu().numpy(), want), name


# ---------------------------------------------------------------- fanouts >= every degree: the masked minibatch
def _grads(m):
    return {k: v.grad.clone() for k, v in named_grads(m) if v.grad is not None}, \
        None if m.embeds is None else m.embeds.grad.clone()


@pytest.mark.parametrize("kind,concat,math,table,identity_dim", [
    ("mean", True, "fp32", "fp32", 0), ("mean", False, "tf32x3", "bf16", 0), ("mean", True, "tf32x3", "fp32", 16),
    ("gcn", False, "fp32", "fp32", 16), ("gcn", False, "tf32x3", "bf16", 0),
    ("maxpool", True, "tf32x3", "fp32", 16), ("maxpool", False, "fp32", "bf16", 0),
    ("meanpool", True, "fp32", "fp32", 0), ("meanpool", False, "tf32x3", "fp32", 16)])
def test_large_fanouts_equal_the_masked_minibatch(gs, kind, concat, math, table, identity_dim):
    m = sup_model(gs, kind, concat, math, table, identity_dim)
    _set_fanouts(m, 256)
    indptr, indices = (dev(a) for a in capped_csr())
    ids = np.array([0, 5, 299, 17, 17, 4, 150, 6, 1, 2, 3, -1], dtype=np.int32)
    labels = np.eye(4, dtype=np.float32)[np.arange(len(ids)) % 4]
    out = []
    for fn in (m.full_neighbor_minibatch_loss, m.sampled_minibatch_loss):
        m.dropout_counter = 40
        m.optimizer.zero_grad(set_to_none=True)
        loss = fn(indptr, indices, ids, labels, dropout=0.5)
        loss.backward()
        out.append((loss.detach(),) + _grads(m) + (m.dropout_counter,))
    assert torch.equal(out[0][0], out[1][0]) and out[0][3] == out[1][3]
    assert set(out[0][1]) == set(out[1][1])
    for k in out[0][1]:
        assert torch.equal(out[0][1][k], out[1][1][k]), k
    assert (out[0][2] is None) == (out[1][2] is None)
    if out[0][2] is not None:
        assert torch.equal(out[0][2], out[1][2])


@pytest.mark.parametrize("kind,identity_dim", [("mean", 16), ("gcn", 0), ("maxpool", 0)])
def test_unsupervised_large_fanouts_equal_the_masked_minibatch(gs, kind, identity_dim):
    m = unsup_model(gs, kind, identity_dim)
    _set_fanouts(m, 256)
    indptr, indices = (dev(a) for a in capped_csr())
    b1, b2 = dev(np.array([1, 2, 3, 9, 40], np.int32)), dev(np.array([4, 4, 38, 0, 299], np.int32))
    neg_state = m.neg_sampler.counter
    out = []
    for fn in (m.full_neighbor_minibatch_loss, m.sampled_minibatch_loss):
        m.dropout_counter, m.neg_sampler.counter = 7, neg_state
        m.optimizer.zero_grad(set_to_none=True)
        loss = fn(indptr, indices, b1, b2, dropout=0.3)
        loss.backward()
        out.append((loss.detach(), [v.grad.clone() for _, v in named_grads_unsup(m)],
                    None if m.embeds is None else m.embeds.grad.clone(), m.dropout_counter))
    assert torch.equal(out[0][0], out[1][0]) and out[0][3] == out[1][3] == 7 + (2 if kind == "maxpool" else 4)
    assert all(torch.equal(a, b) for a, b in zip(out[0][1], out[1][1]))
    if identity_dim:
        assert torch.equal(out[0][2], out[1][2])


# ---------------------------------------------------------------- small fanouts: against the CPU oracle
@pytest.mark.parametrize("kind,concat,math,identity_dim,layers,fanout", [
    ("mean", True, "fp32", 0, 2, 5), ("gcn", False, "fp32", 16, 2, 10), ("maxpool", True, "tf32x3", 0, 2, 3),
    ("meanpool", False, "fp32", 16, 2, 25), ("mean", False, "tf32x3", 16, 3, 4), ("mean", True, "fp32", 16, 1, 1)])
def test_supervised_loss_and_gradients_match_the_oracle(gs, kind, concat, math, identity_dim, layers, fanout):
    m = sup_model(gs, kind, concat, math, "fp32", identity_dim, layers, fanout=fanout)
    indptr, indices = edge_csr(np.random.RandomState(1), 300, 300)
    ids = np.array([0, 5, 299, 17, 17, 4, 150, 6, 1, 2, 3, -1], dtype=np.int32)
    labels = np.eye(4, dtype=np.float32)[np.arange(len(ids)) % 4]
    sampler = m.layer_infos[0].neigh_sampler
    call = sampler.counter
    m.dropout_counter = 13
    feats = m.features.float().cpu().numpy()
    m.optimizer.zero_grad(set_to_none=True)
    loss = m.sampled_minibatch_loss(dev(indptr), dev(indices), ids, labels, dropout=0.4)
    loss.backward()
    assert sampler.counter == call + 1 and m.dropout_counter == 13 + len(fd.site_plan(kind, layers, True))
    fanouts = [info.num_samples for info in m.layer_infos]
    rl, grads, head, demb = sbd.sampled_loss_grads_dropout(
        feats, indptr, indices, oracle_aggs(m), concat, ids, labels, m.node_pred_vars["weights"].detach().cpu().numpy(),
        m.node_pred_vars["bias"].detach().cpu().numpy(), fanouts, sampler.seed, call,
        fd.sites(kind, layers, True, m.dropout_key, 13, 0.4), False, m.weight_decay, identity_dim)
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


# ---------------------------------------------------------------- batch independence, determinism, rates, host reads
def test_a_node_gets_the_same_layer0_row_in_any_batch(gs):
    indptr, indices = graph("rmat")
    N = len(indptr) - 1
    x = torch.randn((N + 1, 32), generator=torch.Generator(device="cuda").manual_seed(5), device="cuda")
    rows = []
    for seeds in ([17, 3, 99], [1000, 17, 5, 6, 7, 8] + list(range(2000, 2500))):
        blocks, offs = gs.ops.csr_blocks(dev(indptr), dev(indices), dev(np.array(seeds, np.int32)), 1, fanouts=[25],
                                         seed=4, call=8, entry_offsets=True)
        b = blocks[0]
        y = gs.ops.csr_aggregate(gs.ops.gather_rows_f32(x, b.src_ids), b.indptr, b.indices, "mean", rows=b.rows,
                                 dropout=((1, 2, 0.5), (1, 3, 0.5), (dev(indptr), b.src_ids, len(indices), offs[0])))
        rows.append(y[seeds.index(17)])
    assert torch.equal(rows[0], rows[1])
    # and it is the whole-graph row over S_0: node 17's entries masked at their global CSR positions
    s_ptr, s_idx = gs.ops.sample_csr_rows(dev(indptr), dev(indices), 25, 4, 8, 0)
    o_ptr, o = sbd.sample_offsets(indptr, 25, 4, 8, 0)
    want = sbd.csr_aggregate_dropout_offsets(x.cpu().numpy(), s_ptr.cpu().numpy(), s_idx.cpu().numpy(), "mean",
                                             (1, 2, 0.5), (1, 3, 0.5), (indptr, None, len(indices), o), [17])
    assert np.array_equal(rows[0].cpu().numpy(), want[0])


def test_determinism_rates_and_host_reads(gs):
    indptr, indices = (dev(a) for a in edge_csr(np.random.RandomState(1), 300, 300))
    ids = dev(np.array([0, 5, 299, 17, 17, 4, 150, 6, 1, 2, 3, -1], dtype=np.int32))
    labels = dev(np.eye(4, dtype=np.float32)[np.arange(12) % 4])

    def run(dropout, steps=2):
        m = sup_model(gs, "mean", True, "fp32", "fp32", 16)
        losses = [m.sampled_minibatch_train_step(indptr, indices, ids, labels, dropout=dropout) for _ in range(steps)]
        return losses, [p.detach().clone() for p in m.parameters()], m.dropout_counter
    none, zero, a, b = run(None), run(0.), run(0.5), run(0.5)
    assert zero[2] == 0 and a[2] == 2 * 5
    for x, y in ((none, zero), (a, b)):
        assert all(torch.equal(p, q) for p, q in zip(x[0] + x[1], y[0] + y[1]))
    assert not torch.equal(none[0][0], a[0][0])
    # the kept fraction of a sampled block's entries
    rmat_ptr, rmat_idx, blk, off = _block_case(gs, "rmat", 100, seed=2)
    ones = torch.ones((blk.src_ids.numel(), 256), device="cuda")
    cnt = torch.diff(blk.indptr)[blk.rows.long().clamp(max=blk.indptr.numel() - 2)]
    y = gs.ops.csr_aggregate(ones, blk.indptr, blk.indices, "mean", rows=blk.rows,
                             dropout=((3, 1, 0.3), (3, 2, 0.3), (dev(rmat_ptr), blk.src_ids, len(rmat_idx), off)))
    has = (cnt > 0) & (blk.rows.long() < blk.indptr.numel() - 1)
    kept = float((y[has] * cnt[has, None].float() * np.float32(0.7)).sum()) / (float(cnt[has].sum()) * 256)
    n_el = float(cnt[has].sum()) * 256
    assert abs(kept - 0.7) < 5 * np.sqrt(0.21 / n_el) + 1e-6, (kept, n_el)
    # the masked call reads back only the block sizes
    m = sup_model(gs, "gcn", False, "fp32", "fp32", 16)
    for dropout in (None, 0.5):                                  # first calls: lazy set-up
        m.sampled_minibatch_loss(indptr, indices, ids, labels, dropout=dropout).backward()
    reads = []
    for dropout in (None, 0.5):
        torch.cuda.synchronize()
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter("always")
            torch.cuda.set_sync_debug_mode("warn")
            try:
                m.sampled_minibatch_loss(indptr, indices, ids, labels, dropout=dropout).backward()
            finally:
                torch.cuda.set_sync_debug_mode("default")
        reads.append(sum("synchroniz" in str(x.message) for x in w))
    print("host synchronisations per sampled loss + backward: dropout None %d, p = 0.5 %d" % tuple(reads))
    assert reads[1] == 1


def test_toy_ppi_epoch_at_half_dropout(gs):
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
    f1, losses = {}, {}
    for path in ("tree", "sampled"):
        gs.inits.manual_seed(3)
        sampler = gs.UniformNeighborSampler(dev(it.adj), seed=1)
        infos = [gs.SAGEInfo("node", sampler, 10, 64), gs.SAGEInfo("node", sampler, 5, 64)]
        m = gs.SupervisedGraphsage(labels.shape[1], {"batch_size": 512, "dropout": 0.5}, feats, dev(it.adj), None, infos,
                                   aggregator_type="mean", sigmoid_loss=True, learning_rate=0.03)
        losses[path] = []
        for i in range(0, len(order), 512):
            b = dev(order[i:i + 512])
            if path == "tree":
                losses[path].append(float(m.train_step(b, d_lab[b.long()])))
            else:
                losses[path].append(float(m.sampled_minibatch_train_step(tr_ptr, tr_idx, b, d_lab[b.long()],
                                                                         dropout=m.dropout_rate)))
        sampler.set_adj(dev(it.test_adj))
        with torch.no_grad():
            pred = m.predict(dev(val)).cpu().numpy()
        f1[path] = calc_f1(labels[val], pred, True)[0]
    s = losses["sampled"]
    print("toy-ppi one epoch of 512-node steps at dropout 0.5: val micro-F1 tree %.4f, sampled blocks %.4f; sampled "
          "loss %.4f -> %.4f over %d steps" % (f1["tree"], f1["sampled"], s[0], s[-1], len(s)))
    assert np.all(np.isfinite(s)) and s[-1] < s[0]
    assert abs(f1["tree"] - f1["sampled"]) <= 0.05
