"""GPU: the models over WeightedNeighborSampler against references on the oracle's draws.  The torch-CPU references of
the existing training tests sample through oracle.torch_ref.sample_padded; here that function serves
oracle/alias_sampling.py's draws instead, so the same references check: supervised loss and gradients (mean, gcn,
maxpool, meanpool; identity_dim 0 and 16; dropout 0 and 0.5), the unsupervised loss and gradients, and the twomaxpool
and seq forwards.  Host-memory, bf16, int8 and fused-pool models give the bits of their device-table twins on the same
weighted draws."""
import numpy as np
import pytest
import torch

from conftest import load_golden, rel_err
from oracle import alias_sampling as al
from oracle import seq as oseq
from oracle import torch_ref
from test_zz_gpu_dropout import _cpu_forward, _cpu_params, _drop_t
from test_zz_gpu_seq import _oracle_aggs
from test_zz_gpu_twomax import _cpu_outputs, _nonzero_biases, _weights
from test_zz_gpu_weighted_sampling import weights_of

pytestmark = pytest.mark.gpu


def _graph():
    """The golden k-hop graph as a CSR (row v = its padded adjacency row) with weights of every kind, and its features."""
    g = load_golden("khop")
    adj, feats = g["adj"], g["feats"]
    N, MD = adj.shape[0] - 1, adj.shape[1]
    indptr = np.arange(N + 1, dtype=np.int64) * MD
    indices = np.ascontiguousarray(adj[:N].reshape(-1)).astype(np.int32)
    return adj, feats, indptr, indices, weights_of(len(indices), "mixed", seed=8)


@pytest.fixture
def weighted(monkeypatch):
    """(adj, feats, sampler factory); torch_ref.sample_padded then draws from the sampler's alias table by the oracle."""
    import graphsage_b200 as gs
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    adj, feats, indptr, indices, w = _graph()
    dev = [torch.from_numpy(x).cuda() for x in (indptr, indices, w)]
    table = gs.ops.csr_alias_table(*dev).cpu().numpy()

    def draws(adj_t, ids_t, k, seed, counter):
        return torch.from_numpy(al.sample(indptr, table, ids_t.numpy(), k, seed, counter))
    monkeypatch.setattr(torch_ref, "sample_padded", draws)
    return adj, feats, lambda seed=123: gs.WeightedNeighborSampler(*dev, seed=seed)


def _supervised(make, adj, feats, kind, concat, rate, d, B=16, C=5, fan=(4, 3), dim=8, **kw):
    import graphsage_b200 as gs
    gs.set_default_math(kw.pop("math", "fp32"))
    gs.inits.manual_seed(5)
    sampler = make()
    sampler.counter = 40
    infos = [gs.SAGEInfo("node", sampler, fan[0], dim), gs.SAGEInfo("node", sampler, fan[1], dim)]
    table = kw.pop("features", None)
    table = torch.from_numpy(feats).cuda() if table is None else table
    m = gs.SupervisedGraphsage(C, {"batch_size": B, "dropout": rate}, table, torch.from_numpy(adj).cuda(), None, infos,
                               concat=concat, aggregator_type=kind, sigmoid_loss=True, learning_rate=0.01,
                               weight_decay=1e-3, identity_dim=d, dropout_seed=555, **kw)
    gen = torch.Generator(device="cuda").manual_seed(2)
    for a in m.aggregators:
        if hasattr(a, "mlp_layers"):
            bias = a.mlp_layers[0].vars["bias"]
            bias.data.add_(torch.randn(bias.shape, generator=gen, device=bias.device) * 0.1)
    return m


@pytest.mark.parametrize("d", [0, 16])
@pytest.mark.parametrize("rate", [0.0, 0.5])
@pytest.mark.parametrize("kind,concat", [("mean", True), ("gcn", False), ("maxpool", True), ("meanpool", False)])
def test_supervised_loss_and_gradients_match_cpu_autograd(weighted, kind, concat, rate, d):
    adj, feats, make = weighted
    rs = np.random.RandomState(5)
    B, C, fan, wd = 16, 5, [4, 3], 1e-3
    m = _supervised(make, adj, feats, kind, concat, rate, d)
    seeds = rs.randint(0, adj.shape[0] - 1, size=B).astype(np.int32)
    seeds[0] = adj.shape[0] - 1                                      # the dummy id draws the dummy
    labels = (rs.rand(B, C) < 0.3).astype(np.float32)
    aggs = _cpu_params(m)
    head = {k: v.detach().cpu().clone().requires_grad_(True) for k, v in m.node_pred_vars.items()}
    E = m.embeds.detach().cpu().clone().requires_grad_(True) if d else None
    table = torch.cat([E, torch.from_numpy(feats)], dim=1) if d else torch.from_numpy(feats)
    out, call = _cpu_forward(adj, table, seeds, fan, aggs, concat, kind, 123, 40, 555, m.dropout_counter, rate)
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
    assert abs(float(loss.detach()) - float(ref.detach())) < 1e-5 * max(1.0, abs(float(ref.detach())))
    for a, ra in zip(m.aggregators, aggs):
        for k in a.vars:
            assert rel_err(a.vars[k].grad.cpu().numpy(), ra[k].grad.numpy(), floor=1e-8) < 2e-4, (kind, k)
        if hasattr(a, "mlp_layers"):
            for k, rk in (("weights", "mlp_weights"), ("bias", "mlp_bias")):
                got = a.mlp_layers[0].vars[k].grad.cpu().numpy()
                want = ra[rk].grad.numpy().reshape(got.shape)
                assert rel_err(got.reshape(1, -1) if k == "bias" else got, want.reshape(1, -1) if k == "bias" else want,
                               floor=1e-8) < 2e-4, (kind, k)
    for k in head:
        assert rel_err(m.node_pred_vars[k].grad.cpu().numpy().reshape(1, -1), head[k].grad.numpy().reshape(1, -1)) < 2e-4
    if d:
        want = E.grad.numpy()
        assert rel_err(m.embeds.grad.cpu().numpy(), want, floor=1e-3 * float(np.abs(want).max())) < 2e-4


def test_unsupervised_loss_and_gradients_match_cpu_autograd(weighted):
    import graphsage_b200 as gs
    import oracle
    adj, feats, make = weighted
    rs = np.random.RandomState(11)
    n, B, NEG = adj.shape[0] - 1, 16, 20
    deg = rs.randint(1, 40, size=n).astype(np.float64)
    b1 = rs.randint(0, n, size=B).astype(np.int32)
    b2 = rs.randint(0, n, size=B).astype(np.int32)
    fan, dim = [5, 3], 12
    gs.set_default_math("fp32")
    sampler = make()
    infos = [gs.SAGEInfo("node", sampler, fan[0], dim), gs.SAGEInfo("node", sampler, fan[1], dim)]
    m = gs.UnsupervisedGraphsage({"batch_size": B, "dropout": 0.}, torch.from_numpy(feats).cuda(),
                                 torch.from_numpy(adj).cuda(), deg, infos, concat=True, aggregator_type="mean",
                                 neg_sample_size=NEG, learning_rate=0.01, weight_decay=1e-3, seed=77)
    aggs = [{k: v.detach().cpu().clone().requires_grad_(True) for k, v in a.vars.items()} for a in m.aggregators]
    neg = oracle.sample_unigram(deg, NEG, 77, 0)
    A, F = torch.from_numpy(adj), torch.from_numpy(feats)
    o1 = torch_ref.forward(A, F, torch.from_numpy(b1), fan, aggs, True, "mean", 123, 0)
    o2 = torch_ref.forward(A, F, torch.from_numpy(b2), fan, aggs, True, "mean", 123, 2)
    on = torch_ref.forward(A, F, torch.from_numpy(neg), fan, aggs, True, "mean", 123, 4)
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
    assert np.isfinite(float(m.train_step(torch.from_numpy(b1), torch.from_numpy(b2))))


@pytest.mark.parametrize("math", ["fp32", "tf32x3"])
def test_twomaxpool_and_seq_forward_match_the_references(weighted, math):
    import graphsage_b200 as gs
    adj, feats, make = weighted
    rs = np.random.RandomState(3)
    B = 32
    seeds = rs.randint(0, adj.shape[0] - 1, size=B).astype(np.int32)
    gs.set_default_math(math)
    try:
        s = make()
        infos = [gs.SAGEInfo("node", s, 10, 64), gs.SAGEInfo("node", s, 5, 64)]
        m = gs.SampleAndAggregate({"batch_size": B, "dropout": 0.}, torch.from_numpy(feats).cuda(),
                                  torch.from_numpy(adj).cuda(), None, infos, concat=True, aggregator_type="twomaxpool")
        m.forward(torch.from_numpy(seeds))
        _nonzero_biases(m)
        c0 = s.counter
        out = m.forward(torch.from_numpy(seeds)).cpu().numpy()
        ref = _cpu_outputs(adj, torch.from_numpy(feats).double(), seeds, [10, 5], _weights(m, torch.float64), True,
                           123, c0)
        assert rel_err(out, ref.detach().numpy() if torch.is_tensor(ref) else ref) < 1e-4
        s = make()
        infos = [gs.SAGEInfo("node", s, 5, 16), gs.SAGEInfo("node", s, 3, 16)]
        m = gs.SampleAndAggregate({"batch_size": B, "dropout": 0.}, torch.from_numpy(feats).cuda(),
                                  torch.from_numpy(adj).cuda(), None, infos, concat=True, aggregator_type="seq")
        m.forward(torch.from_numpy(seeds))
        c0 = s.counter
        out = m.forward(torch.from_numpy(seeds), normalize=False).cpu().numpy()
        samples = [seeds] + _draws(s, seeds, [3, 5], c0)
        ref = oseq.aggregate_khop_seq(samples, feats, [5, 3], [1, 3, 15], B, _oracle_aggs(m.aggregators), True,
                                      dtype=np.float64)
        assert rel_err(out, ref) < 1e-4
    finally:
        gs.set_default_math("fp32")


def _draws(sampler, seeds, fanouts, counter):
    return al.sample_khop(sampler.indptr.cpu().numpy(), sampler.table.cpu().numpy(), seeds, fanouts, sampler.seed,
                          counter)


@pytest.mark.parametrize("variant", ["host-fp32", "host-bf16", "int8", "fused-host-fp32"])
def test_tables_give_the_device_table_bits_on_the_same_draws(weighted, variant):
    import graphsage_b200 as gs
    adj, feats, make = weighted
    x = feats.copy()
    kind, math, kw = ("maxpool", "bf16", {"fused_pool": True}) if variant.startswith("fused") else ("mean", "fp32", {})
    if variant == "int8":
        table = gs.Int8Features(x, device="cuda")
        twin_table = table.dequantize()
    elif variant == "host-bf16":
        table = gs.HostFeatures(torch.from_numpy(x).to(torch.bfloat16))
        twin_table = torch.from_numpy(x).to(torch.bfloat16).cuda()
    else:
        table = gs.HostFeatures(x)
        twin_table = torch.from_numpy(x).cuda()
    try:
        m = _supervised(make, adj, feats, kind, True, 0.0, 0, math=math, features=table, **kw)
        twin = _supervised(make, adj, feats, kind, True, 0.0, 0, math=math, features=twin_table, **kw)
        rs = np.random.RandomState(6)
        for step in range(4):
            ids = torch.from_numpy(rs.randint(0, adj.shape[0] - 1, size=16).astype(np.int32))
            lab = torch.from_numpy((rs.rand(16, 5) < 0.3).astype(np.float32))
            assert torch.equal(m.train_step(ids, lab), twin.train_step(ids, lab)), step
        assert torch.equal(m.predict(ids), twin.predict(ids))
    finally:
        gs.set_default_math("fp32")
