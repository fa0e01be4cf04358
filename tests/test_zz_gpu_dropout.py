"""GPU: training dropout (reference aggregators.py:46-47 / 104-105, layers.py:107, supervised_models.py:88-90) under the
Philox mask contract of oracle/dropout.py.

The three kernels against the oracle (gs_dropout_apply bit for bit, gs_gather_mean_dropout, the masked embedding gradient),
the supervised and unsupervised losses and gradients against torch-CPU autograd on the oracle's masks, bit-reproducible
clipped-Adam training, the evaluation paths of a model built with dropout, and the refused combinations."""
import numpy as np
import pytest
import torch

from conftest import load_golden, rel_err
from oracle import dropout as od
from oracle import torch_ref

pytestmark = pytest.mark.gpu


def _np_drop(x, site, scale=1.0, group=1, rows=None):
    seed, call, rate = site
    x = np.asarray(x, np.float32)
    rows = x.shape[0] * group if rows is None else rows
    xr = np.repeat(x, group, axis=0)[:rows]
    m = od.keep_mask(seed, call, rate, np.arange(rows), x.shape[1])
    return np.where(m, (xr * np.float32(scale)) / od.keep_prob(rate), np.float32(0)).astype(np.float32)


# ---------------------------------------------------------------------------------------------------- gs_dropout_apply
@pytest.mark.parametrize("F", [1, 5, 130, 602])
@pytest.mark.parametrize("group,scale,accumulate", [(1, 1.0, False), (3, 0.25, True), (10, 1.0 / 11, False)])
def test_dropout_apply_is_bit_identical_to_the_oracle(F, group, scale, accumulate):
    import graphsage_b200 as gs
    rs = np.random.RandomState(F + group)
    n = 257
    base = torch.from_numpy(rs.randn(n, F + 3).astype(np.float32)).cuda()
    x = base[:, :F]                                                      # strided rows
    site = (2 ** 40 + 17, 9, 0.37)
    rows = n * group - (1 if group > 1 else 0)
    out0 = rs.randn(rows, F + 5).astype(np.float32)
    out = torch.from_numpy(out0).cuda()[:, 2:2 + F]
    gs.ops.dropout_apply(x, site, rows=rows, group=group, scale=scale, out=out, accumulate=accumulate)
    want = _np_drop(x.cpu().numpy(), site, scale, group, rows)
    if accumulate:
        want = out0[:, 2:2 + F] + want
    assert np.array_equal(out.cpu().numpy(), want)
    full = torch.from_numpy(out0).cuda()
    gs.ops.dropout_apply(x, site, rows=rows, group=group, scale=scale, out=full[:, 2:2 + F], accumulate=accumulate)
    assert np.array_equal(full[:, :2].cpu().numpy(), out0[:, :2]) and np.array_equal(full[:, 2 + F:].cpu().numpy(), out0[:, 2 + F:])


def test_dropout_apply_rate_zero_in_place_and_refusals():
    import graphsage_b200 as gs
    x = torch.randn(100, 33, device="cuda")
    assert torch.equal(gs.ops.dropout_apply(x, (1, 2, 0.0)), x)
    y = x.clone()
    gs.ops.dropout_apply(y, (1, 2, 0.5), out=y)
    assert torch.equal(y, gs.ops.dropout_apply(x, (1, 2, 0.5)))
    for bad in (-0.5, 1.0, float("nan")):
        with pytest.raises(ValueError):
            gs.ops.dropout_apply(x, (1, 2, bad))


# ---------------------------------------------------------------------------------------------------- gs_gather_mean_dropout
def _oracle_gather(src, segs, nsites, ssites, include_self):
    src = src.cpu().numpy()
    rows = max(s.out_row0 + s.n for s in segs)
    F = src.shape[1]
    xs, xm = np.zeros((rows, F), np.float32), np.zeros((rows, F), np.float32)
    for s, ns, ss in zip(segs, nsites, ssites):
        n, k = s.n, s.k
        nid = s.neigh_ids[:n * k].cpu().numpy() if s.neigh_ids is not None else s.neigh_row0 + np.arange(n * k)
        sid = s.self_ids[:n].cpu().numpy() if s.self_ids is not None else s.self_row0 + np.arange(n)
        nb = _np_drop(src[nid], ns).reshape(n, k, F)
        sv = _np_drop(src[sid], ss)
        acc = np.zeros((n, F), np.float32)
        for j in range(k):
            acc += nb[:, j]
        if include_self:
            acc += sv
        xm[s.out_row0:s.out_row0 + n] = acc / np.float32(k + (1 if include_self else 0))
        xs[s.out_row0:s.out_row0 + n] = sv
    return xs, xm


@pytest.mark.parametrize("F,pitch", [(602, 608), (50, 56), (37, 37), (1300, 1304)])
@pytest.mark.parametrize("include_self", [False, True])
@pytest.mark.parametrize("addressing", ["ids", "rows"])
def test_gather_mean_dropout_matches_the_oracle(F, pitch, include_self, addressing):
    import graphsage_b200 as gs
    rs = np.random.RandomState(F + int(include_self))
    N = 700
    table = torch.from_numpy(rs.randn(N, pitch).astype(np.float32)).cuda()[:, :F]
    if addressing == "ids":
        s0 = torch.from_numpy(rs.randint(0, N, size=13).astype(np.int32)).cuda()
        s1 = torch.from_numpy(rs.randint(0, N, size=13 * 5).astype(np.int32)).cuda()
        s2 = torch.from_numpy(rs.randint(0, N, size=13 * 5 * 3).astype(np.int32)).cuda()
        segs = [gs.ops.Seg(13, 5, self_ids=s0, neigh_ids=s1, out_row0=0),
                gs.ops.Seg(65, 3, self_ids=s1, neigh_ids=s2, out_row0=13)]
    else:
        segs = [gs.ops.Seg(13, 5, self_row0=0, neigh_row0=13, out_row0=0), gs.ops.Seg(65, 3, self_row0=13, neigh_row0=78,
                                                                                       out_row0=13)]
    nsites = [(5, 0, 0.5), (5, 2, 0.1)]
    ssites = [(5, 1, 0.5), (5, 3, 0.1)]
    xs, xm = gs.ops.gather_mean_dropout(table, segs, nsites, ssites, include_self=include_self, want_self=True)
    ws, wm = _oracle_gather(table, segs, nsites, ssites, include_self)
    assert np.array_equal(xs[:, :F].cpu().numpy(), ws)
    assert rel_err(xm[:, :F].cpu().numpy(), wm) < 1e-5
    assert float(xm[:, F:].abs().sum()) == 0 and float(xs[:, F:].abs().sum()) == 0
    # rate 0 is the plain fused gather, bit for bit
    z = [(5, 0, 0.0)] * 2
    zs, zm = gs.ops.gather_mean_dropout(table, segs, z, z, include_self=include_self)
    ps, pm = gs.ops.gather_mean(table, segs, include_self=include_self, want_self=True)
    assert torch.equal(zs, ps) and torch.equal(zm, pm)


def test_gather_mean_dropout_full_layer0_size():
    """configs[1] layer 0: 512 seeds, fanout 25 x 10, 602 columns (128,000 masked neighbour rows in the hop-2 segment)."""
    import graphsage_b200 as gs
    rs = np.random.RandomState(1)
    N, F, B = 20000, 602, 512
    table = torch.from_numpy(rs.randn(N, 608).astype(np.float32)).cuda()[:, :F]
    s0 = torch.from_numpy(rs.randint(0, N, size=B).astype(np.int32)).cuda()
    s1 = torch.from_numpy(rs.randint(0, N, size=B * 25).astype(np.int32)).cuda()
    s2 = torch.from_numpy(rs.randint(0, N, size=B * 250).astype(np.int32)).cuda()
    segs = [gs.ops.Seg(B, 25, self_ids=s0, neigh_ids=s1, out_row0=0), gs.ops.Seg(B * 25, 10, self_ids=s1, neigh_ids=s2,
                                                                                 out_row0=B)]
    nsites, ssites = [(77, 0, 0.5), (77, 2, 0.5)], [(77, 1, 0.5), (77, 3, 0.5)]
    xs, xm = gs.ops.gather_mean_dropout(table, segs, nsites, ssites)
    ws, wm = _oracle_gather(table, segs, nsites, ssites, False)
    assert np.array_equal(xs[:, :F].cpu().numpy(), ws)
    assert rel_err(xm[:, :F].cpu().numpy(), wm) < 1e-5


# ---------------------------------------------------------------------------------------------------- masked embedding gradient
def test_masked_embedding_grad_matches_fp64_index_add_and_is_reproducible():
    import graphsage_b200 as gs
    rs = np.random.RandomState(4)
    n_rows, d, n, k = 3001, 64, 400, 25
    self_ids = torch.from_numpy(rs.randint(0, n_rows, size=n).astype(np.int32)).cuda()
    neigh_ids = torch.from_numpy(rs.randint(0, 50, size=n * k).astype(np.int32)).cuda()     # long runs
    gs_ = torch.from_numpy(rs.randn(n, d + 4).astype(np.float32)).cuda()[:, :d]
    gm = torch.from_numpy(rs.randn(n, d).astype(np.float32)).cuda()
    lists = [(self_ids, gs_, 1, 1.0), (neigh_ids, gm, k, 1.0 / k)]
    sites = [(9, 1, 0.5), (9, 0, 0.3)]
    out = gs.ops.embedding_grad(lists, n_rows, d, sites=sites)
    ref = torch.zeros((n_rows, d), dtype=torch.float64)
    for (ids, g, group, scale), (seed, call, rate) in zip(lists, sites):
        m = ids.numel()
        rows = g.double().cpu().repeat_interleave(group, dim=0)[:m] * scale
        mask = torch.from_numpy(od.keep_mask(seed, call, rate, np.arange(m), d))
        rows = torch.where(mask, rows / float(od.keep_prob(rate)), torch.zeros((), dtype=torch.float64))
        ref.index_add_(0, ids.long().cpu(), rows)
    assert rel_err(out.double().cpu().numpy(), ref.numpy(), floor=1e-6) < 1e-5
    assert torch.equal(out, gs.ops.embedding_grad(lists, n_rows, d, sites=sites))
    zero = gs.ops.embedding_grad(lists, n_rows, d, sites=[(9, 0, 0.0)] * 2)
    assert torch.equal(zero, gs.ops.embedding_grad(lists, n_rows, d))


# ---------------------------------------------------------------------------------------------------- the models
def _mask_t(site, rows, F):
    seed, call, rate = site
    return torch.from_numpy(od.keep_mask(seed, call, rate, np.arange(rows), F)).float()


def _drop_t(x, site):
    return x / float(od.keep_prob(site[2])) * _mask_t(site, x.shape[0], x.shape[1])


def _cpu_forward(adj, table, seeds, fan, aggs, concat, kind, seed, counter, key, call, rate):
    """The oracle's op sequence with dropout (sites in the reference's call order from `call`) in torch autograd.
    Returns (l2-normalised outputs, next call)."""
    adj_t = torch.from_numpy(adj)
    L = len(fan)
    samples = [torch.from_numpy(seeds)]
    for k in range(L):
        samples.append(torch_ref.sample_padded(adj_t, samples[k], fan[L - k - 1], seed, counter + k).reshape(-1))
    hidden = [table.index_select(0, s.long()) for s in samples]
    for layer in range(L):
        a, last, nxt = aggs[layer], layer == L - 1, []
        for hop in range(L - layer):
            k = fan[L - hop - 1]
            neigh, selfv = hidden[hop + 1], hidden[hop]
            n, F = selfv.shape
            if kind in ("mean", "gcn"):
                nb = _drop_t(neigh, (key, call, rate)).reshape(n, k, F)
                sv = _drop_t(selfv, (key, call + 1, rate))
                call += 2
                if kind == "gcn":
                    y = torch.cat([nb, sv[:, None]], dim=1).mean(dim=1) @ a["weights"]
                else:
                    fs, fn = sv @ a["self_weights"], nb.mean(dim=1) @ a["neigh_weights"]
                    y = torch.cat([fs, fn], dim=1) if concat else fs + fn
            else:
                xn = _drop_t(neigh, (key, call, rate))
                call += 1
                h = torch.relu(xn @ a["mlp_weights"] + a["mlp_bias"]).reshape(n, k, -1)
                hp = h.amax(dim=1) if kind == "maxpool" else h.mean(dim=1)
                fs, fn = selfv @ a["self_weights"], hp @ a["neigh_weights"]
                y = torch.cat([fs, fn], dim=1) if concat else fs + fn
            nxt.append(y if last else torch.relu(y))
        hidden = nxt
    out = hidden[0]
    return out / torch.sqrt(torch.clamp((out * out).sum(dim=1, keepdim=True), min=1e-12)), call


def _cpu_params(m):
    aggs = []
    for a in m.aggregators:
        p = {k: v.detach().cpu().clone().requires_grad_(True) for k, v in a.vars.items()}
        if hasattr(a, "mlp_layers"):
            p["mlp_weights"] = a.mlp_layers[0].vars["weights"].detach().cpu().clone().requires_grad_(True)
            p["mlp_bias"] = a.mlp_layers[0].vars["bias"].detach().cpu().clone().requires_grad_(True)
        aggs.append(p)
    return aggs


def _supervised(kind, concat, rate, d=0, B=16, C=5, fan=(4, 3), dim=8, seed=123, counter=40, dropout_seed=555, lr=0.01):
    import graphsage_b200 as gs
    g = load_golden("khop")
    adj, feats = g["adj"], g["feats"]
    gs.set_default_math("fp32")
    sampler = gs.UniformNeighborSampler(torch.from_numpy(adj).cuda(), seed=seed)
    sampler.counter = counter
    infos = [gs.SAGEInfo("node", sampler, fan[0], dim), gs.SAGEInfo("node", sampler, fan[1], dim)]
    m = gs.SupervisedGraphsage(C, {"batch_size": B, "dropout": rate}, torch.from_numpy(feats).cuda(), torch.from_numpy(adj).cuda(),
                               None, infos, concat=concat, aggregator_type=kind, sigmoid_loss=True, learning_rate=lr,
                               weight_decay=1e-3, identity_dim=d, dropout_seed=dropout_seed)
    gen = torch.Generator(device="cuda").manual_seed(2)      # the same non-zero MLP bias for models built alike
    for a in m.aggregators:
        if hasattr(a, "mlp_layers"):
            bias = a.mlp_layers[0].vars["bias"]
            bias.data.add_(torch.randn(bias.shape, generator=gen, device=bias.device) * 0.1)
    return m, adj, feats


KINDS = [("mean", True), ("mean", False), ("gcn", False), ("maxpool", True), ("meanpool", False)]


@pytest.mark.parametrize("d", [0, 6])
@pytest.mark.parametrize("rate", [0.1, 0.5])
@pytest.mark.parametrize("kind,concat", KINDS)
def test_supervised_dropout_loss_and_gradients_match_cpu_autograd(kind, concat, rate, d):
    rs = np.random.RandomState(5)
    B, C, fan, wd = 16, 5, [4, 3], 1e-3
    m, adj, feats = _supervised(kind, concat, rate, d=d)
    n = adj.shape[0] - 1
    seeds = rs.randint(0, n, size=B).astype(np.int32)
    labels = (rs.rand(B, C) < 0.3).astype(np.float32)
    aggs = _cpu_params(m)
    head = {k: v.detach().cpu().clone().requires_grad_(True) for k, v in m.node_pred_vars.items()}
    E = m.embeds.detach().cpu().clone().requires_grad_(True) if d else None
    table = torch.cat([E, torch.from_numpy(feats)], dim=1) if d else torch.from_numpy(feats)
    call0 = m.dropout_counter
    out, call = _cpu_forward(adj, table, seeds, fan, aggs, concat, kind, 123, 40, 555, call0, rate)
    logits = _drop_t(out, (555, call, rate)) @ head["weights"] + head["bias"]
    ref = torch.nn.functional.binary_cross_entropy_with_logits(logits, torch.from_numpy(labels))
    for a in aggs:
        for k in ("neigh_weights", "self_weights", "weights", "bias"):
            if k in a:
                ref = ref + wd * 0.5 * (a[k] * a[k]).sum()
    for v in head.values():
        ref = ref + wd * 0.5 * (v * v).sum()
    ref.backward()
    loss = m.loss(torch.from_numpy(seeds), torch.from_numpy(labels), dropout=rate)
    loss.backward()
    assert m.dropout_counter == call + 1
    assert abs(float(loss) - float(ref)) < 1e-5 * max(1.0, abs(float(ref)))
    for a, ra in zip(m.aggregators, aggs):
        for k in a.vars:
            assert rel_err(a.vars[k].grad.cpu().numpy(), ra[k].grad.numpy(), floor=1e-8) < 2e-4, (kind, k)
        if hasattr(a, "mlp_layers"):
            for k, rk in (("weights", "mlp_weights"), ("bias", "mlp_bias")):
                got = a.mlp_layers[0].vars[k].grad.cpu().numpy().reshape(1, -1) if k == "bias" else \
                    a.mlp_layers[0].vars[k].grad.cpu().numpy()
                want = ra[rk].grad.numpy().reshape(got.shape)
                assert rel_err(got, want, floor=1e-8) < 2e-4, (kind, k)
    for k in head:
        assert rel_err(m.node_pred_vars[k].grad.cpu().numpy().reshape(1, -1), head[k].grad.numpy().reshape(1, -1)) < 2e-4
    if d:
        # an embedding row sums many masked contributions; rows whose terms cancel are judged against 1e-3 of the largest
        # gradient entry, the scale of their fp32 rounding
        want = E.grad.numpy()
        assert rel_err(m.embeds.grad.cpu().numpy(), want, floor=1e-3 * float(np.abs(want).max())) < 2e-4


@pytest.mark.parametrize("kind,concat", KINDS)
def test_unsupervised_dropout_three_passes_match_cpu_autograd(kind, concat):
    import graphsage_b200 as gs
    import oracle
    g = load_golden("khop")
    rs = np.random.RandomState(11)
    adj, feats = g["adj"], g["feats"]
    n, B, NEG, rate = adj.shape[0] - 1, 16, 20, 0.5
    deg = rs.randint(1, 40, size=n).astype(np.float64)
    b1 = rs.randint(0, n, size=B).astype(np.int32)
    b2 = rs.randint(0, n, size=B).astype(np.int32)
    fan, dim = [5, 3], 12
    gs.set_default_math("fp32")
    sampler = gs.UniformNeighborSampler(torch.from_numpy(adj).cuda(), seed=123)
    infos = [gs.SAGEInfo("node", sampler, fan[0], dim), gs.SAGEInfo("node", sampler, fan[1], dim)]
    m = gs.UnsupervisedGraphsage({"batch_size": B, "dropout": rate}, torch.from_numpy(feats).cuda(),
                                 torch.from_numpy(adj).cuda(), deg, infos, concat=concat, aggregator_type=kind,
                                 neg_sample_size=NEG, learning_rate=0.01, weight_decay=1e-3, seed=77, dropout_seed=31)
    for a in m.aggregators:
        if hasattr(a, "mlp_layers"):
            a.mlp_layers[0].vars["bias"].data.add_(torch.randn_like(a.mlp_layers[0].vars["bias"]) * 0.1)
    aggs = _cpu_params(m)
    table = torch.from_numpy(feats)
    neg = oracle.sample_unigram(deg, NEG, 77, 0)
    o1, call = _cpu_forward(adj, table, b1, fan, aggs, concat, kind, 123, 0, 31, 0, rate)
    o2, call = _cpu_forward(adj, table, b2, fan, aggs, concat, kind, 123, 2, 31, call, rate)
    on, call = _cpu_forward(adj, table, np.asarray(neg, np.int32), fan, aggs, concat, kind, 123, 4, 31, call, rate)
    ref = torch.nn.functional.softplus(-(o1 * o2).sum(1)).sum() + torch.nn.functional.softplus(o1 @ on.t()).sum()
    for a in aggs:
        for k in ("neigh_weights", "self_weights", "weights", "bias"):
            if k in a:
                ref = ref + 1e-3 * 0.5 * (a[k] * a[k]).sum()
    ref = ref / B
    ref.backward()
    loss = m.loss(torch.from_numpy(b1), torch.from_numpy(b2), dropout=rate)
    loss.backward()
    assert m.dropout_counter == call
    assert abs(float(loss.detach()) - float(ref.detach())) < 1e-5 * max(1.0, abs(float(ref.detach())))
    for a, ra in zip(m.aggregators, aggs):
        for k in a.vars:
            assert rel_err(a.vars[k].grad.cpu().numpy(), ra[k].grad.numpy(), floor=1e-8) < 2e-4, k
        if hasattr(a, "mlp_layers"):
            assert rel_err(a.mlp_layers[0].vars["weights"].grad.cpu().numpy(), ra["mlp_weights"].grad.numpy(),
                           floor=1e-8) < 2e-4


# ---------------------------------------------------------------------------------------------------- training and evaluation
def _train(kind, dropout_seed, steps=5, rate=0.5):
    import graphsage_b200 as gs
    gs.inits.manual_seed(11)
    m, adj, _ = _supervised(kind, True if kind != "gcn" else False, rate, d=4, B=32, fan=(5, 3), dim=16, seed=7, counter=0,
                            dropout_seed=dropout_seed)
    rs = np.random.RandomState(9)
    n = adj.shape[0] - 1
    for _ in range(steps):
        seeds = rs.randint(0, n, size=32).astype(np.int32)
        labels = (rs.rand(32, 5) < 0.3).astype(np.float32)
        assert np.isfinite(float(m.train_step(torch.from_numpy(seeds), torch.from_numpy(labels))))
    return [p.detach().clone() for p in m.parameters()], m


@pytest.mark.parametrize("kind", ["mean", "maxpool"])
def test_dropout_training_is_bit_reproducible_and_keyed_by_the_seed(kind):
    a, ma = _train(kind, 1000)
    b, _ = _train(kind, 1000)
    c, _ = _train(kind, 1001)
    assert ma.dropout_counter > 0
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    assert not all(torch.equal(x, y) for x, y in zip(a, c))


@pytest.mark.parametrize("kind", ["mean", "gcn", "maxpool"])
def test_evaluation_paths_of_a_dropout_model_do_not_drop(kind):
    import graphsage_b200 as gs
    concat = kind != "gcn"
    gs.inits.manual_seed(3)
    md, adj, _ = _supervised(kind, concat, 0.5)
    gs.inits.manual_seed(3)
    m0, _, _ = _supervised(kind, concat, 0.0)
    for p, q in zip(md.parameters(), m0.parameters()):
        assert torch.equal(p, q)
    rs = np.random.RandomState(2)
    seeds = torch.from_numpy(rs.randint(0, adj.shape[0] - 1, size=16).astype(np.int32))
    labels = torch.from_numpy((rs.rand(16, 5) < 0.3).astype(np.float32))
    assert torch.equal(md.predict(seeds), m0.predict(seeds))
    assert torch.equal(md.forward(seeds), m0.forward(seeds))
    assert torch.equal(md.loss(seeds, labels, dropout=0.), m0.loss(seeds, labels))
    assert md.dropout_counter == 0 and md.dropout_rate == 0.5
    assert all(a.dropout == 0 for a in md.aggregators)


def test_refused_dropout_combinations():
    import graphsage_b200 as gs
    from graphsage_b200 import supervised_models as sm
    for bad in (-0.1, 1.0, 2.0):
        with pytest.raises(ValueError):
            _supervised("mean", True, bad)
    g = load_golden("khop")
    sampler = gs.UniformNeighborSampler(torch.from_numpy(g["adj"]).cuda(), seed=1)
    infos = [gs.SAGEInfo("node", sampler, 3, 8), gs.SAGEInfo("node", sampler, 2, 8)]
    bf16 = torch.from_numpy(g["feats"]).cuda().to(torch.bfloat16)
    with pytest.raises(NotImplementedError):
        gs.SupervisedGraphsage(3, {"batch_size": 4, "dropout": 0.5}, bf16, torch.from_numpy(g["adj"]).cuda(), None, infos,
                               aggregator_type="mean")

    class _Sharded(object):
        c_table = None

    with pytest.raises(NotImplementedError):
        sm.refuse_dropout_table(_Sharded())
    m, _, _ = _supervised("mean", True, 0.0)
    with pytest.raises(ValueError):
        m.loss(torch.zeros(4, dtype=torch.int32), torch.zeros(4, 5), dropout=1.0)
