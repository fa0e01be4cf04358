"""GPU: trainable node embeddings (identity_dim > 0; reference supervised_models.py:51-67, models.py:229-245).

The embedding-gradient kernel (ops.embedding_grad) against an fp64 index_add_, the layer-0 backward of every aggregator
against torch-CPU autograd on the oracle's op sequence over concat([E, X]) (or E alone), clipped-Adam training, the
forward paths on the trained table, training from a dataset without features, and the refused combinations."""
import numpy as np
import pytest
import torch

from conftest import load_golden, rel_err
from oracle import torch_ref

pytestmark = pytest.mark.gpu


# ---------------------------------------------------------------------------------------------------- the kernel
def _ref_grad(lists, n_rows, d):
    out = torch.zeros((n_rows, d), dtype=torch.float64)
    mag = torch.zeros((n_rows, d), dtype=torch.float64)
    for ids, grad, group, scale in lists:
        ids = ids.reshape(-1).long().cpu()
        n = ids.numel()
        if n == 0:
            continue
        rows = grad[:(n + group - 1) // group, :d].double().cpu().repeat_interleave(group, dim=0)[:n] * scale
        ok = (ids >= 0) & (ids < n_rows)
        out.index_add_(0, ids[ok], rows[ok])
        mag.index_add_(0, ids[ok], rows[ok].abs())
    return out, mag


def _check_grad(got, lists, n_rows, d):
    ref, mag = _ref_grad(lists, n_rows, d)
    got = got.double().cpu()
    assert got.shape == ref.shape
    untouched = mag.sum(dim=1) == 0
    assert torch.equal(got[untouched], torch.zeros_like(got[untouched]))          # rows nobody addresses are exactly zero
    num = (got - ref).norm(dim=1)
    # 1e-5 relative per row; a row whose terms cancel to under 1% of their absolute sum (d = 1 rows do) is judged against
    # 1% of that sum - no fp32 summation order can keep the relative error of a near-cancelling sum small
    den = torch.maximum(ref.norm(dim=1), 1e-2 * mag.norm(dim=1))
    assert float((num[~untouched] / den[~untouched]).max()) < 1e-5


def _strided(rows, d, rs, extra=0):
    """float32 CUDA [rows, d] view with row stride d + extra (extra > 0: a strided view into a wider buffer)."""
    base = torch.from_numpy(rs.randn(rows, d + extra).astype(np.float32)).cuda()
    return base[:, :d]


def _ids(rs, n, n_rows, pad_frac=0.1):
    ids = rs.randint(0, n_rows - 1, size=n).astype(np.int32)
    ids[rs.rand(n) < pad_frac] = n_rows - 1                                        # the padding id N
    return torch.from_numpy(ids).cuda()


def _segment_lists(form, rs, n, k, n_rows, d, extra):
    """One hop segment's lists in the layer-0 backward's form (mean / gcn / pool)."""
    self_ids, neigh_ids = _ids(rs, n, n_rows), _ids(rs, n * k, n_rows)
    if form == "mean":
        return [(self_ids, _strided(n, d, rs, extra), 1, 1.0), (neigh_ids, _strided(n, d, rs, extra), k, 1.0 / k)]
    if form == "gcn":
        g = _strided(n, d, rs, extra)
        return [(self_ids, g, 1, 1.0 / (k + 1)), (neigh_ids, g, k, 1.0 / (k + 1))]
    return [(self_ids, _strided(n, d, rs, extra), 1, 1.0), (neigh_ids, _strided(n * k, d, rs, extra), 1, 1.0)]


@pytest.mark.parametrize("d", [1, 50, 64, 128])
@pytest.mark.parametrize("form", ["mean", "gcn", "pool"])
def test_embedding_grad_matches_fp64_index_add(form, d):
    import graphsage_b200 as gs
    rs = np.random.RandomState(d + len(form))
    n_rows = 3001
    lists = _segment_lists(form, rs, 40, 10, n_rows, d, extra=3 if d % 2 else 0) + \
        _segment_lists(form, rs, 400, 25, n_rows, d, extra=7)
    out = gs.ops.embedding_grad(lists, n_rows, d)
    _check_grad(out, lists, n_rows, d)
    again = gs.ops.embedding_grad(lists, n_rows, d)
    assert torch.equal(out, again)                                                   # deterministic, bit for bit


def test_embedding_grad_long_runs_duplicates_and_edges():
    """One id repeated 60,000 times (a long run split over many chunks), the padding id, runs that straddle chunk edges,
    ids outside [0, n_rows) (ignored), all eight lists, an empty list."""
    import graphsage_b200 as gs
    rs = np.random.RandomState(3)
    n_rows, d = 5000, 64
    hub = np.full(60000, 1234, np.int32)
    hub[::7] = n_rows - 1
    mixed = rs.randint(0, 40, size=20000).astype(np.int32)                           # few ids: runs of ~500 each
    odd = rs.randint(0, n_rows, size=333).astype(np.int32)
    odd[:3] = [-1, n_rows, 2 ** 31 - 1]
    lists = [(torch.from_numpy(hub).cuda(), _strided(60000 // 4, d, rs, 5), 4, 0.25),
             (torch.from_numpy(mixed).cuda(), _strided(20000, d, rs), 1, 1.0),
             (torch.from_numpy(odd).cuda(), _strided(333, d, rs), 1, -2.0),
             (torch.zeros(0, dtype=torch.int32, device="cuda"), _strided(1, d, rs), 1, 1.0)]
    lists += [(_ids(rs, 1000, n_rows), _strided(100, d, rs), 10, 0.1) for _ in range(4)]
    out = gs.ops.embedding_grad(lists, n_rows, d)
    _check_grad(out, lists, n_rows, d)
    assert torch.equal(out, gs.ops.embedding_grad(lists, n_rows, d))


def test_embedding_grad_no_contributions_and_strided_out():
    import graphsage_b200 as gs
    out = torch.full((17, 5), 7.0, device="cuda")
    gs.ops.embedding_grad([], 17, 5, out=out)
    assert torch.equal(out, torch.zeros_like(out))
    empty = [(torch.zeros(0, dtype=torch.int32, device="cuda"), torch.zeros((0, 5), device="cuda"), 1, 1.0)]
    assert torch.equal(gs.ops.embedding_grad(empty, 17, 5), torch.zeros((17, 5), device="cuda"))
    rs = np.random.RandomState(1)
    lists = [(_ids(rs, 900, 17), _strided(300, 5, rs, 2), 3, 0.5)]
    wide = torch.full((17, 12), 3.0, device="cuda")
    gs.ops.embedding_grad(lists, 17, 5, out=wide[:, 2:7])                             # row stride 12
    _check_grad(wide[:, 2:7], lists, 17, 5)
    assert torch.equal(wide[:, :2], torch.full((17, 2), 3.0, device="cuda"))
    assert torch.equal(wide[:, 7:], torch.full((17, 5), 3.0, device="cuda"))


def test_embedding_grad_full_size():
    """Reddit shape: N = 232,965, batch 512, fanout 25 x 10, d = 64 - 138,752 contributions in four lists (mean form)."""
    import graphsage_b200 as gs
    rs = np.random.RandomState(7)
    n_rows, d, B = 232966, 64, 512
    lists = _segment_lists("mean", rs, B, 10, n_rows, d, extra=64) + _segment_lists("mean", rs, B * 10, 25, n_rows, d, extra=64)
    assert sum(ids.numel() for ids, _, _, _ in lists) == 138752
    out = gs.ops.embedding_grad(lists, n_rows, d)
    _check_grad(out, lists, n_rows, d)
    assert torch.equal(out, gs.ops.embedding_grad(lists, n_rows, d))


# ---------------------------------------------------------------------------------------------------- the model
def _cpu_outputs(adj, table, seeds, fan, aggs, concat, kind, seed, counter):
    """The oracle's op sequence (torch_ref) on an arbitrary input table; the pooling aggregators restated here."""
    if kind in ("mean", "gcn"):
        return torch_ref.forward(torch.from_numpy(adj), table, torch.from_numpy(seeds), fan, aggs, concat, kind, seed, counter)
    adj_t, seeds_t = torch.from_numpy(adj), torch.from_numpy(seeds)
    L = len(fan)
    samples, sup = [seeds_t], 1
    for k in range(L):
        t = L - k - 1
        sup *= fan[t]
        samples.append(torch_ref.sample_padded(adj_t, samples[k], fan[t], seed, counter + k).reshape(-1))
    hidden = [table.index_select(0, s.long()) for s in samples]
    for layer in range(L):
        a, last, nxt = aggs[layer], layer == L - 1, []
        for hop in range(L - layer):
            k = fan[L - hop - 1]
            neigh, selfv = hidden[hop + 1], hidden[hop]
            n = selfv.shape[0]
            h = torch.relu(neigh @ a["mlp_weights"] + a["mlp_bias"]).reshape(n, k, -1)
            hp = h.amax(dim=1) if kind == "maxpool" else h.mean(dim=1)
            fs, fn = selfv @ a["self_weights"], hp @ a["neigh_weights"]
            y = torch.cat([fs, fn], dim=1) if concat else fs + fn
            nxt.append(y if last else torch.relu(y))
        hidden = nxt
    out = hidden[0]
    return out / torch.sqrt(torch.clamp((out * out).sum(dim=1, keepdim=True), min=1e-12))


def _cpu_params(m):
    aggs = []
    for a in m.aggregators:
        p = {k: v.detach().cpu().clone().requires_grad_(True) for k, v in a.vars.items()}
        if hasattr(a, "mlp_layers"):
            p["mlp_weights"] = a.mlp_layers[0].vars["weights"].detach().cpu().clone().requires_grad_(True)
            p["mlp_bias"] = a.mlp_layers[0].vars["bias"].detach().cpu().clone().requires_grad_(True)
        aggs.append(p)
    return aggs


def _cpu_table(E, feats, with_features):
    return torch.cat([E, torch.from_numpy(feats)], dim=1) if with_features else E


def _supervised(kind, concat, with_features, d, B, C, fan, dim, seed=123, counter=40, lr=0.01, wd=1e-3):
    import graphsage_b200 as gs
    g = load_golden("khop")
    adj, feats = g["adj"], g["feats"]
    gs.set_default_math("fp32")
    sampler = gs.UniformNeighborSampler(torch.from_numpy(adj).cuda(), seed=seed)
    sampler.counter = counter
    infos = [gs.SAGEInfo("node", sampler, fan[0], dim), gs.SAGEInfo("node", sampler, fan[1], dim)]
    m = gs.SupervisedGraphsage(C, {"batch_size": B, "dropout": 0.}, torch.from_numpy(feats).cuda() if with_features else None,
                               torch.from_numpy(adj).cuda(), None, infos, concat=concat, aggregator_type=kind,
                               sigmoid_loss=True, learning_rate=lr, weight_decay=wd, identity_dim=d)
    for a in m.aggregators:                              # a non-zero MLP bias so its gradient path is exercised
        if hasattr(a, "mlp_layers"):
            a.mlp_layers[0].vars["bias"].data.add_(torch.randn_like(a.mlp_layers[0].vars["bias"]) * 0.1)
    return m, adj, feats, sampler


@pytest.mark.parametrize("with_features", [True, False])
@pytest.mark.parametrize("kind,concat", [("mean", True), ("mean", False), ("gcn", False), ("maxpool", True),
                                         ("meanpool", False)])
def test_identity_loss_and_gradients_match_cpu_autograd(kind, concat, with_features):
    rs = np.random.RandomState(5)
    B, C, fan, dim, d, wd = 16, 5, [4, 3], 8, 6, 1e-3
    m, adj, feats, _ = _supervised(kind, concat, with_features, d, B, C, fan, dim, wd=wd)
    n = adj.shape[0] - 1
    assert m.dims[0] == d + (feats.shape[1] if with_features else 0)
    assert tuple(m.embeds.shape) == (n + 1, d) and any(p is m.embeds for p in m.parameters())
    assert all(p is not m.embeds for p in m.decayed_parameters())
    seeds = rs.randint(0, n, size=B).astype(np.int32)
    seeds[0] = 3                                          # an isolated node: its samples are the padding id N
    labels = (rs.rand(B, C) < 0.3).astype(np.float32)
    aggs = _cpu_params(m)
    head = {k: v.detach().cpu().clone().requires_grad_(True) for k, v in m.node_pred_vars.items()}
    E = m.embeds.detach().cpu().clone().requires_grad_(True)
    out = _cpu_outputs(adj, _cpu_table(E, feats, with_features), seeds, fan, aggs, concat, kind, 123, 40)
    ref = torch.nn.functional.binary_cross_entropy_with_logits(out @ head["weights"] + head["bias"], torch.from_numpy(labels))
    for a in aggs:                                        # weight decay: aggregator vars and head only, never the embeddings
        for k in ("neigh_weights", "self_weights", "weights", "bias"):
            if k in a:
                ref = ref + wd * 0.5 * (a[k] * a[k]).sum()
    for v in head.values():
        ref = ref + wd * 0.5 * (v * v).sum()
    ref.backward()
    loss = m.loss(torch.from_numpy(seeds), torch.from_numpy(labels))
    loss.backward()
    assert abs(float(loss) - float(ref)) < 1e-5 * max(1.0, abs(float(ref)))
    for a, ra in zip(m.aggregators, aggs):
        for k in a.vars:
            assert rel_err(a.vars[k].grad.cpu().numpy(), ra[k].grad.numpy(), floor=1e-8) < 2e-4, (kind, k)
        if hasattr(a, "mlp_layers"):
            assert rel_err(a.mlp_layers[0].vars["weights"].grad.cpu().numpy(), ra["mlp_weights"].grad.numpy(), floor=1e-8) < 2e-4
    for k in head:
        assert rel_err(m.node_pred_vars[k].grad.cpu().numpy().reshape(1, -1), head[k].grad.numpy().reshape(1, -1)) < 2e-4
    assert float(E.grad[n].abs().sum()) > 0               # the padding row is trained like any other
    assert rel_err(m.embeds.grad.cpu().numpy(), E.grad.numpy(), floor=1e-8) < 2e-4


def test_identity_unsupervised_loss_and_gradients_match_cpu():
    import graphsage_b200 as gs
    import oracle
    g = load_golden("khop")
    rs = np.random.RandomState(11)
    adj, feats = g["adj"], g["feats"]
    n, B, NEG, d = adj.shape[0] - 1, 16, 20, 8
    deg = rs.randint(1, 40, size=n).astype(np.float64)
    b1 = rs.randint(0, n, size=B).astype(np.int32)
    b2 = rs.randint(0, n, size=B).astype(np.int32)
    fan, dim = [5, 3], 12
    gs.set_default_math("fp32")
    sampler = gs.UniformNeighborSampler(torch.from_numpy(adj).cuda(), seed=123)
    infos = [gs.SAGEInfo("node", sampler, fan[0], dim), gs.SAGEInfo("node", sampler, fan[1], dim)]
    m = gs.UnsupervisedGraphsage({"batch_size": B, "dropout": 0.}, torch.from_numpy(feats).cuda(),
                                 torch.from_numpy(adj).cuda(), deg, infos, concat=True, aggregator_type="mean",
                                 neg_sample_size=NEG, learning_rate=0.01, weight_decay=1e-3, seed=77, identity_dim=d)
    assert any(p is m.embeds for p in m.parameters()) and all(p is not m.embeds for p in m.decayed_parameters())
    aggs = _cpu_params(m)
    E = m.embeds.detach().cpu().clone().requires_grad_(True)
    table = _cpu_table(E, feats, True)
    A = torch.from_numpy(adj)
    neg = oracle.sample_unigram(deg, NEG, 77, 0)
    o1 = torch_ref.forward(A, table, torch.from_numpy(b1), fan, aggs, True, "mean", 123, 0)
    o2 = torch_ref.forward(A, table, torch.from_numpy(b2), fan, aggs, True, "mean", 123, 2)
    on = torch_ref.forward(A, table, torch.from_numpy(neg), fan, aggs, True, "mean", 123, 4)
    ref = torch.nn.functional.softplus(-(o1 * o2).sum(1)).sum() + torch.nn.functional.softplus(o1 @ on.t()).sum()
    for a in aggs:
        for v in a.values():
            ref = ref + 1e-3 * 0.5 * (v * v).sum()
    ref = ref / B
    ref.backward()
    loss = m.loss(torch.from_numpy(b1), torch.from_numpy(b2))
    loss.backward()
    assert abs(float(loss.detach()) - float(ref.detach())) < 1e-5 * max(1.0, abs(float(ref.detach())))
    for a, ra in zip(m.aggregators, aggs):
        for k in a.vars:
            assert rel_err(a.vars[k].grad.cpu().numpy(), ra[k].grad.numpy(), floor=1e-8) < 3e-4, k
    assert rel_err(m.embeds.grad.cpu().numpy(), E.grad.numpy(), floor=1e-8) < 3e-4
    assert np.isfinite(float(m.train_step(torch.from_numpy(b1), torch.from_numpy(b2))))


def _train_identity(kind, steps, rs_seed=9):
    import graphsage_b200 as gs
    gs.inits.manual_seed(11)                              # the same initial table and weights on every call
    B, C, fan, dim, d = 32, 5, [5, 3], 16, 8
    m, adj, feats, sampler = _supervised(kind, True, True, d, B, C, fan, dim, seed=7, counter=0, wd=0.0)
    rs = np.random.RandomState(rs_seed)
    n = adj.shape[0] - 1
    batches = []
    for _ in range(steps):
        seeds = rs.randint(0, n, size=B).astype(np.int32)
        seeds[0] = 3                                      # an isolated node: its samples are the padding id N
        batches.append((seeds, (rs.rand(B, C) < 0.3).astype(np.float32)))
    return m, adj, feats, sampler, batches, fan


def test_identity_training_tracks_cpu_adam_and_is_bit_reproducible():
    """Five clipped-Adam steps follow the same steps on the CPU restatement, the embedding table (dummy row included) too;
    a second identical run ends with a bit-identical table."""
    m, adj, feats, _, batches, fan = _train_identity("mean", 5)
    aggs = _cpu_params(m)
    head = {k: v.detach().cpu().clone().requires_grad_(True) for k, v in m.node_pred_vars.items()}
    E = m.embeds.detach().cpu().clone().requires_grad_(True)
    E0 = E.detach().clone()
    params = [v for a in aggs for v in a.values()] + list(head.values()) + [E]
    opt = torch.optim.Adam(params, lr=0.01)
    gpu_losses, cpu_losses = [], []
    for step, (seeds, labels) in enumerate(batches):
        gpu_losses.append(float(m.train_step(torch.from_numpy(seeds), torch.from_numpy(labels))))
        opt.zero_grad()
        out = _cpu_outputs(adj, _cpu_table(E, feats, True), seeds, fan, aggs, True, "mean", 7, 2 * step)
        ref = torch.nn.functional.binary_cross_entropy_with_logits(out @ head["weights"] + head["bias"],
                                                                   torch.from_numpy(labels))
        ref.backward()
        for p in params:
            p.grad.clamp_(-5.0, 5.0)
        opt.step()
        cpu_losses.append(float(ref))
    assert np.allclose(gpu_losses, cpu_losses, rtol=2e-3), (gpu_losses, cpu_losses)
    for a, ra in zip(m.aggregators, aggs):
        for k in a.vars:
            assert rel_err(a.vars[k].detach().cpu().numpy(), ra[k].detach().numpy()) < 5e-3
    got = m.embeds.detach().cpu()
    moved = (E.detach() != E0).any(dim=1)
    assert bool(moved[-1])                                                     # the dummy row N was sampled and trained
    assert rel_err(got.numpy(), E.detach().numpy()) < 5e-3
    assert torch.equal(got[~moved], E0[~moved])                                # rows never sampled: bit-identical
    m2, _, _, _, batches2, _ = _train_identity("mean", 5)
    for seeds, labels in batches2:
        m2.train_step(torch.from_numpy(seeds), torch.from_numpy(labels))
    assert torch.equal(m2.embeds.detach(), m.embeds.detach())
    assert torch.equal(m2.features.detach(), m.features.detach())


def test_forward_paths_see_the_trained_table():
    """After training, eager forward(), a CUDA-graph runner captured before the last step, and the bf16 max-pool forward
    (whose bf16 cast of the table is cached per tensor version) all read the updated embeddings."""
    import graphsage_b200 as gs
    m, adj, feats, sampler, batches, fan = _train_identity("mean", 4)
    for seeds, labels in batches[:3]:
        m.train_step(torch.from_numpy(seeds), torch.from_numpy(labels))
    seeds = torch.from_numpy(batches[0][0])
    sampler.counter = 100
    runner = m.graphed(seeds.numel())
    m.train_step(torch.from_numpy(batches[3][0]), torch.from_numpy(batches[3][1]))     # after capture
    runner.reset(0)
    out_g = runner(seeds.cuda()).detach().clone()
    sampler.counter = 100
    with torch.no_grad():
        out_e = m.forward(seeds)
    runner.close()
    aggs = _cpu_params(m)
    table = _cpu_table(m.embeds.detach().cpu(), feats, True)
    ref = _cpu_outputs(adj, table, batches[0][0], fan, aggs, True, "mean", 7, 100).detach()
    assert rel_err(out_e.cpu().numpy(), ref.numpy()) < 1e-4
    assert rel_err(out_g.cpu().numpy(), out_e.cpu().numpy()) < 1e-6
    # ---- max-pool: the bf16 K4 forward caches the table's bf16 cast per version; a training step must refresh it
    mp, adj, feats, sampler, batches, fan = _train_identity("maxpool", 2)

    def bf16_forward(counter):
        for a in mp.aggregators:
            a.math = gs.ops.MATH_BF16
        sampler.counter = counter
        try:
            with torch.no_grad():
                return mp.forward(torch.from_numpy(batches[0][0]))
        finally:
            for a in mp.aggregators:
                a.math = gs.ops.MATH_FP32_SIMT
    before = bf16_forward(200)
    for seeds, labels in batches:
        mp.train_step(torch.from_numpy(seeds), torch.from_numpy(labels))
    cached = bf16_forward(200)
    mp.aggregators[0]._bf16_ref = None                                          # force a fresh cast
    fresh = bf16_forward(200)
    assert torch.equal(cached, fresh) and not torch.equal(cached, before)
    ref = _cpu_outputs(adj, _cpu_table(mp.embeds.detach().cpu(), feats, True), batches[0][0], fan, _cpu_params(mp), True,
                       "maxpool", 7, 200).detach()
    assert rel_err(cached.cpu().numpy(), ref.numpy()) < 5e-2                   # bf16 operands


def test_reference_fixture_forward_on_the_gpu():
    """tests/golden/identity.npz: the reference's constructor + aggregate(); our model with the fixture's table and
    weights reproduces its output, with features and without."""
    import graphsage_b200 as gs
    g = load_golden("identity")
    adj, feats, seeds, fan, d = g["adj"], g["feats"], g["seeds"], [int(x) for x in g["fanout"]], int(g["identity_dim"])
    gs.set_default_math("fp32")
    for tag in ("feat", "nofeat"):
        key = "sup_%s_" % tag
        sampler = gs.UniformNeighborSampler(torch.from_numpy(adj).cuda(), seed=123)
        infos = [gs.SAGEInfo("node", sampler, fan[i], int(g[key + "L%d_self_weights" % i].shape[1])) for i in range(2)]
        m = gs.SampleAndAggregate({"batch_size": len(seeds), "dropout": 0.},
                                  torch.from_numpy(feats).cuda() if tag == "feat" else None, torch.from_numpy(adj).cuda(),
                                  None, infos, concat=True, aggregator_type="mean", identity_dim=d)
        assert m.dims == [int(x) for x in g[key + "dims"]]
        m.forward(torch.from_numpy(seeds))                                     # creates the aggregators
        with torch.no_grad():
            m.embeds.copy_(torch.from_numpy(g[key + "embeds"]))
            for li, a in enumerate(m.aggregators):
                for k in a.vars:
                    a.vars[k].copy_(torch.from_numpy(g["%sL%d_%s" % (key, li, k)]))
        np.testing.assert_array_equal(m.features.cpu().numpy(), g[key + "features"])
        sampler.counter = 40
        with torch.no_grad():
            out = m.forward(torch.from_numpy(seeds), normalize=False)
        assert rel_err(out.cpu().numpy(), g[key + "out"]) < 1e-5


def test_featureless_dataset_trains(tmp_path):
    """A dataset written without a feature file loads with feats None; SupervisedGraphsage(features=None,
    identity_dim=16) trains on it: finite loss, the rows of sampled ids move, every other row stays bit-identical."""
    import graphsage_b200 as gs
    from graphsage_b200 import minibatch, utils
    from graphsage_b200.graph import Graph
    r = np.random.RandomState(2)
    n = 400
    G = Graph()
    for u in range(n):
        G.add_node(u, val=bool(u % 10 == 1), test=bool(u % 10 == 2))
    for u in range(n - 20):                                           # the last 20 nodes stay isolated
        for v in r.choice(n - 20, size=3, replace=False):
            if int(v) != u:
                G.add_edge(u, int(v))
    for u, v in G.edges():
        G[u][v]["train_removed"] = bool(G.node[u]["val"] or G.node[v]["val"] or G.node[u]["test"] or G.node[v]["test"])
    id_map = {u: u for u in range(n)}
    class_map = {u: int(u % 3) for u in range(n)}
    prefix = str(tmp_path / "bare")
    utils.write_dataset(prefix, G, None, id_map, class_map)
    G2, feats, id_map2, _, class_map2 = utils.load_data(prefix)
    assert feats is None
    np.random.seed(123)
    it = minibatch.NodeMinibatchIterator(G2, id_map2, None, class_map2, 3, batch_size=24, max_degree=8)
    adj = torch.from_numpy(it.adj.astype(np.int32)).cuda()
    gs.set_default_math("fp32")
    sampler = gs.UniformNeighborSampler(adj, seed=5)
    infos = [gs.SAGEInfo("node", sampler, 5, 16), gs.SAGEInfo("node", sampler, 3, 16)]
    m = gs.SupervisedGraphsage(3, {"batch_size": 24, "dropout": 0.}, None, adj, None, infos, concat=True,
                               aggregator_type="mean", sigmoid_loss=False, learning_rate=0.01, identity_dim=16)
    assert m.dims[0] == 16 and tuple(m.embeds.shape) == (adj.shape[0], 16)
    E0 = m.embeds.detach().clone()
    touched = torch.zeros(adj.shape[0], dtype=torch.bool, device="cuda")
    for _ in range(4):
        feed, labels = it.next_minibatch_feed_dict()
        batch = torch.as_tensor(np.asarray(feed["batch"]), dtype=torch.int32)
        c0 = sampler.counter
        loss = m.train_step(batch, torch.as_tensor(np.asarray(labels), dtype=torch.float32))
        assert np.isfinite(float(loss))
        c1, sampler.counter = sampler.counter, c0                      # the ids this step sampled
        samples, _ = m.sample(batch.cuda(), m.layer_infos, batch_size=batch.numel())
        sampler.counter = c1
        for s in samples:
            touched[s.long()] = True
    changed = (m.embeds.detach() != E0).any(dim=1)
    assert bool(changed[touched].all())
    assert torch.equal(m.embeds.detach()[~touched], E0[~touched]) and int((~touched).sum()) > 0


def test_refused_combinations():
    import graphsage_b200 as gs
    g = load_golden("khop")
    adj, feats = torch.from_numpy(g["adj"]).cuda(), torch.from_numpy(g["feats"]).cuda()
    sampler = gs.UniformNeighborSampler(adj, seed=1)
    infos = [gs.SAGEInfo("node", sampler, 3, 8), gs.SAGEInfo("node", sampler, 2, 8)]
    ph = {"batch_size": 4, "dropout": 0.}

    class ShardedStub(object):                      # what SampleAndAggregate recognises a node-partitioned table by
        shape = tuple(feats.shape)

        def c_table(self):
            raise AssertionError("not reached")

    with pytest.raises(NotImplementedError):
        gs.SupervisedGraphsage(3, ph, ShardedStub(), adj, None, infos, identity_dim=4)
    with pytest.raises(NotImplementedError):
        gs.SupervisedGraphsage(3, ph, feats, adj, None, infos, identity_dim=4, distributed=True)
    with pytest.raises(NotImplementedError):
        gs.UnsupervisedGraphsage(ph, feats, adj, np.ones(adj.shape[0] - 1), infos, identity_dim=4, distributed=True)
    with pytest.raises(NotImplementedError):
        gs.SampleAndAggregate(ph, feats.to(torch.bfloat16), adj, None, infos, identity_dim=4)
    with pytest.raises(ValueError):
        gs.SampleAndAggregate(ph, None, adj, None, infos, identity_dim=0)
    with pytest.raises(ValueError):                  # features and adjacency must both have N+1 rows
        gs.SampleAndAggregate(ph, feats[:-1], adj, None, infos, identity_dim=4)
