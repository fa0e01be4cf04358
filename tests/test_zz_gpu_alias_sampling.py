"""GPU: fixed-fanout draws in proportion to edge weight (WeightedNeighborSampler).  The alias tables byte for byte
against oracle/alias_sampling.py on toy-ppi, an R-MAT graph with a 10^5-entry row, a row of 10^6 entries, an edgeless
graph and E = 0, every weight kind; gs_sample_alias and _khop byte for byte (1 - 4 hops, fanouts 1 .. 1024, ids out of
range, the dummy, more draws than one pass of the capped grid), counter_dev, determinism; the law on 2^20 copies of one
row and the sampled-mean estimator; and the models over the sampler: forward against the oracle's aggregation on the
oracle's draws, the graphed forward and training step against eager twins across a set_graph swap, the per-hop
fallback and a few training steps on toy-ppi."""
import numpy as np
import pytest
import torch

from oracle import aggregate as oagg
from oracle import alias_sampling as al
from test_zz_gpu_full_neighbor import dev
from test_zz_gpu_sampled_blocks import graph
from test_zz_gpu_weighted_sampling import KINDS, weights_of

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def gs():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    import graphsage_b200
    graphsage_b200._lib.lib()
    return graphsage_b200


def _graph(name):
    if name in ("toy-ppi", "rmat"):
        return graph(name)
    if name == "million":
        rs = np.random.RandomState(3)
        deg = np.array([5, 1000000, 0, 3], np.int64)
        indptr = np.concatenate([[0], np.cumsum(deg)]).astype(np.int64)
        return indptr, rs.randint(0, 4, size=int(indptr[-1])).astype(np.int32)
    if name == "edgeless":
        return np.zeros(40, np.int64), np.zeros(0, np.int32)
    if name == "zero-nodes":
        return np.zeros(1, np.int64), np.zeros(0, np.int32)
    raise ValueError(name)


def _table(gs, indptr, indices, w):
    return gs.ops.csr_alias_table(dev(indptr), dev(indices), dev(w))


CASES = ([("toy-ppi", k) for k in ("heavy", "mixed")] + [("rmat", k) for k in KINDS]
         + [("million", "heavy"), ("million", "mixed"), ("edgeless", "positive"), ("zero-nodes", "positive")])


@pytest.mark.parametrize("name,kind", CASES)
def test_table_bit_exact(gs, name, kind):
    indptr, indices = _graph(name)
    w = weights_of(len(indices), kind, seed=len(indices) % 97)
    got = _table(gs, indptr, indices, w)
    torch.cuda.synchronize()
    assert got.shape == (len(indices), 4) and got.dtype == torch.int32
    assert np.array_equal(got.cpu().numpy(), al.build_table(indptr, indices, w))


@pytest.mark.parametrize("k", [1, 10, 25, 64, 1024])
def test_draws_bit_exact(gs, k):
    indptr, indices = graph("rmat")
    N = len(indptr) - 1
    w = weights_of(len(indices), "mixed", seed=2)
    tab = _table(gs, indptr, indices, w)
    rs = np.random.RandomState(k)
    n = max(20, 600000 // k)                                      # past one pass of the capped grid
    ids = rs.randint(0, N, size=n).astype(np.int32)
    ids[:6] = [-1, N, N + 4, 17, 17, 0]
    got = gs.ops.sample_alias(dev(indptr), tab, dev(ids), k, 99, 5)
    want = al.sample(indptr, tab.cpu().numpy(), ids, k, 99, 5)
    assert np.array_equal(got.cpu().numpy(), want)


@pytest.mark.parametrize("fanouts,n_seeds", [([1], 300), ([25], 300), ([10, 25], 300), ([64, 3], 300), ([3, 1, 4], 300),
                                             ([2, 3, 2, 5], 300), ([25, 10], 2000)])
def test_khop_equals_successive_calls(gs, fanouts, n_seeds):
    indptr, indices = graph("toy-ppi")
    N = len(indptr) - 1
    w = weights_of(len(indices), "heavy", seed=1)
    tab = _table(gs, indptr, indices, w)
    # 2000 seeds at (25, 10): 550,000 elements, past one pass of the capped grid (132 SMs x 8 CTAs x 256 threads)
    seeds = np.concatenate([np.random.RandomState(0).randint(0, N, n_seeds), [-2, N, N + 1]]).astype(np.int32)
    got = gs.ops.sample_alias_khop(dev(indptr), tab, dev(seeds), fanouts, 7, 11)
    want = al.sample_khop(indptr, tab.cpu().numpy(), seeds, fanouts, 7, 11)
    for g, x in zip(got, want):
        assert np.array_equal(g.cpu().numpy(), x)
    # the device counter word adds to the host counter
    cdev = torch.tensor([6], dtype=torch.int64, device="cuda")
    got2 = gs.ops.sample_alias_khop(dev(indptr), tab, dev(seeds), fanouts, 7, 5, counter_dev=cdev)
    for g, x in zip(got2, want):
        assert np.array_equal(g.cpu().numpy(), x)
    one = gs.ops.sample_alias(dev(indptr), tab, dev(seeds), fanouts[0], 7, 5, counter_dev=cdev)
    assert np.array_equal(one.reshape(-1).cpu().numpy(), want[0])


def test_repeated_calls_are_byte_identical_and_a_new_counter_differs(gs):
    indptr, indices = graph("toy-ppi")
    w = weights_of(len(indices), "positive")
    tab = _table(gs, indptr, indices, w)
    assert torch.equal(tab, _table(gs, indptr, indices, w))
    ids = dev(np.arange(0, len(indptr) - 1, 3, dtype=np.int32))
    a = gs.ops.sample_alias(dev(indptr), tab, ids, 10, 1, 0)
    assert torch.equal(a, gs.ops.sample_alias(dev(indptr), tab, ids, 10, 1, 0))
    assert not torch.equal(a, gs.ops.sample_alias(dev(indptr), tab, ids, 10, 1, 1))


@pytest.mark.parametrize("kind", ["heavy", "mixed"])
def test_law_on_many_copies_of_one_row(gs, kind):
    d = 40
    indptr = np.array([0, d], np.int64)
    indices = np.arange(d, dtype=np.int32)
    w = weights_of(d, kind, seed=9)
    tab = _table(gs, indptr, indices, w)
    n = 1 << 20
    got = gs.ops.sample_alias(dev(indptr), tab, dev(np.zeros(n, np.int32)), 1, 3, 0).reshape(-1)
    cnt = np.bincount(got.cpu().numpy(), minlength=d + 1)
    law, den = al.alias_law(tab.cpu().numpy(), indptr, 0)
    for u in range(d + 1):
        p = law.get(u, 0) / den
        sd = np.sqrt(n * p * (1 - p))
        assert abs(cnt[u] - n * p) <= 5 * sd + 1e-9, (u, cnt[u], n * p)


def test_sampled_mean_estimates_the_weighted_mean(gs):
    rs = np.random.RandomState(2)
    N, F, k, reps = 30, 8, 25, 400
    deg = rs.randint(1, 60, size=N)
    indptr = np.concatenate([[0], np.cumsum(deg)]).astype(np.int64)
    indices = rs.randint(0, N, size=int(indptr[-1])).astype(np.int32)
    w = weights_of(len(indices), "heavy", seed=4)
    x = rs.randn(N + 1, F).astype(np.float64)
    x[N] = 0
    tab = _table(gs, indptr, indices, w)
    ids = dev(np.tile(np.arange(N, dtype=np.int32), reps))
    s = gs.ops.sample_alias(dev(indptr), tab, ids, k, 8, 0).cpu().numpy().reshape(reps, N, k)
    est = x[s].mean(axis=2)                                              # [reps, N, F]
    for v in range(N):
        a, z = indptr[v], indptr[v + 1]
        wv = w[a:z].astype(np.float64)
        mean = (wv[:, None] * x[indices[a:z]]).sum(0) / wv.sum()
        var = (wv[:, None] * (x[indices[a:z]] - mean) ** 2).sum(0) / wv.sum()
        se = np.sqrt(var / (k * reps)) + 1e-12
        assert (np.abs(est[:, v].mean(0) - mean) <= 5 * se + 1e-9).all(), v


def _model(gs, sampler, feats, kind, math, fan=(25, 10), cls=None, dropout=0.0, identity_dim=0, concat=True):
    gs.set_default_math(math)
    gs.inits.manual_seed(3)
    infos = [gs.SAGEInfo("node", sampler, fan[0], 16), gs.SAGEInfo("node", sampler, fan[1], 16)]
    adj = torch.zeros((feats.shape[0], 1), dtype=torch.int32, device="cuda")
    if cls is None:
        m = gs.SampleAndAggregate({"batch_size": 48, "dropout": dropout}, feats, adj, None, infos, concat=concat,
                                  aggregator_type=kind, identity_dim=identity_dim)
    else:
        m = gs.SupervisedGraphsage(cls, {"batch_size": 48, "dropout": dropout}, feats, adj, None, infos, concat=concat,
                                   aggregator_type=kind, learning_rate=0.01, identity_dim=identity_dim)
    return m


def _aggs(model, kind):
    out = []
    for a in model.aggregators:
        d = dict(type=kind, **{k: v.detach().cpu().numpy() for k, v in a.vars.items()})
        if kind == "maxpool":
            d.update(mlp_weights=a.mlp_layers[0].vars["weights"].detach().cpu().numpy(),
                     mlp_bias=a.mlp_layers[0].vars["bias"].detach().cpu().numpy())
        out.append(d)
    return out


@pytest.mark.parametrize("kind,math", [("mean", "fp32"), ("mean", "tf32x3"), ("gcn", "fp32"), ("gcn", "tf32x3"),
                                       ("maxpool", "fp32"), ("maxpool", "tf32x3")])
def test_forward_matches_the_oracle_on_the_oracle_draws(gs, kind, math):
    indptr, indices = graph("toy-ppi")
    N = len(indptr) - 1
    w = weights_of(len(indices), "mixed", seed=3)
    rs = np.random.RandomState(0)
    feats = np.vstack([rs.randn(N, 50), np.zeros((1, 50))]).astype(np.float32)
    s = gs.WeightedNeighborSampler(dev(indptr), dev(indices), dev(w), seed=21)
    concat = kind != "gcn"                                        # GCN has no self half (reference models.py)
    m = _model(gs, s, torch.from_numpy(feats).cuda(), kind, math, concat=concat)
    seeds = rs.randint(0, N, 48).astype(np.int32)
    try:
        out = m.forward(dev(seeds), normalize=True).cpu().numpy()
    finally:
        gs.set_default_math("fp32")
    samples = [seeds] + al.sample_khop(indptr, s.table.cpu().numpy(), seeds, [10, 25], 21, 0)
    ref = oagg.aggregate_khop(samples, feats, [25, 10], [1, 10, 250], 48, _aggs(m, kind), concat)
    ref = ref / np.sqrt(np.maximum((ref.astype(np.float64) ** 2).sum(1, keepdims=True), 1e-12))
    assert np.abs(out - ref).max() <= 1e-4 * max(1.0, np.abs(ref).max())
    assert s.counter == 2


def test_per_hop_fallback_matches_the_per_hop_oracle(gs):
    indptr, indices = graph("toy-ppi")
    N = len(indptr) - 1
    w = weights_of(len(indices), "heavy", seed=3)
    s = gs.WeightedNeighborSampler(dev(indptr), dev(indices), dev(w), seed=4)
    feats = torch.zeros((N + 1, 8), device="cuda")
    m = _model(gs, s, feats, "mean", "fp32", fan=(70, 3))
    seeds = np.arange(0, 96, 2, dtype=np.int32)
    samples, _ = m.sample(dev(seeds), m.layer_infos)
    want = al.sample_khop(indptr, s.table.cpu().numpy(), seeds, [3, 70], 4, 0)
    for g, x in zip(samples[1:], want):
        assert np.array_equal(g.cpu().numpy(), x)


def test_graphed_forward_and_train_step_match_eager_twins_across_a_graph_swap(gs):
    indptr, indices = graph("toy-ppi")
    N = len(indptr) - 1
    w = dev(weights_of(len(indices), "heavy", seed=5))
    w2 = dev(weights_of(len(indices), "positive", seed=6))
    rs = np.random.RandomState(1)
    feats = torch.from_numpy(np.vstack([rs.randn(N, 24), np.zeros((1, 24))]).astype(np.float32)).cuda()
    ip, ix = dev(indptr), dev(indices)
    sa, sb = (gs.WeightedNeighborSampler(ip, ix, w, seed=2) for _ in range(2))
    batches = [dev(rs.randint(0, N, 48).astype(np.int32)) for _ in range(4)]
    ma = _model(gs, sa, feats, "mean", "fp32")
    ma.forward(batches[0])                         # the aggregators are made on the first forward, from the seeded RNG
    mb = _model(gs, sb, feats, "mean", "fp32")
    mb.forward(batches[0])
    runner = gs.models.GraphedForward(ma, 48)
    tab = sa.table
    for i, b in enumerate(batches):
        with _no_host_sync():
            got = runner(b).clone()
        want = mb.forward(b)
        assert torch.equal(got, want), i
        sa.set_graph(ip, ix, w2)                   # another graph in between, then back: no rebuild
        sa.set_graph(ip, ix, w)
        assert sa.table is tab
    runner.close()
    # a graphed training step replays the eager twin's losses
    C = 5
    ta, tb = (_model(gs, s, feats, "mean", "fp32", cls=C) for s in (gs.WeightedNeighborSampler(ip, ix, w, seed=8),
                                                                      gs.WeightedNeighborSampler(ip, ix, w, seed=8)))
    labels = torch.zeros((48, C), device="cuda")
    labels[torch.arange(48), torch.from_numpy(rs.randint(0, C, 48))] = 1
    gs.make_adam_capturable(tb.optimizer)
    step = ta.graphed_train_step(48)
    s_train, t_tab = ta.layer_infos[0].neigh_sampler, ta.layer_infos[0].neigh_sampler.table
    for i, b in enumerate(batches + [batches[0][:20]]):
        if b.numel() == 48:
            with _no_host_sync():
                loss = step(b, labels)
        else:                                        # a short last batch runs eagerly between replays
            loss = ta.train_step(b, labels[:20])
        assert torch.equal(loss, tb.train_step(b, labels[:b.numel()])), i
        s_train.set_graph(ip, ix, w2)                # another graph in between, then back: the captured table is kept
        s_train.set_graph(ip, ix, w)
        assert s_train.table is t_tab
    step2 = step(batches[1], labels)
    assert torch.equal(step2, tb.train_step(batches[1], labels))


class _no_host_sync(object):
    """torch raises on any synchronising CUDA call made inside (a replay must not wait for the device)."""

    def __enter__(self):
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")

    def __exit__(self, *exc):
        torch.cuda.set_sync_debug_mode("default")
        return False


def test_training_steps_on_toy_ppi_reduce_the_loss(gs):
    indptr, indices = graph("toy-ppi")
    N = len(indptr) - 1
    w = dev(weights_of(len(indices), "heavy", seed=7))
    rs = np.random.RandomState(4)
    C = 6
    y = rs.randint(0, C, N)
    feats = np.vstack([np.eye(C)[y] + 0.3 * rs.randn(N, C), np.zeros((1, C))]).astype(np.float32)
    s = gs.WeightedNeighborSampler(dev(indptr), dev(indices), w, seed=1)
    m = _model(gs, s, torch.from_numpy(feats).cuda(), "mean", "fp32", cls=C)
    b = dev(rs.randint(0, N, 48).astype(np.int32))
    labels = torch.from_numpy(np.eye(C)[y[b.cpu().numpy()]].astype(np.float32)).cuda()
    first = float(m.loss(b, labels).detach())
    for _ in range(30):
        m.train_step(b, labels)
    assert float(m.loss(b, labels).detach()) < first


def test_argument_errors(gs):
    indptr, indices = graph("toy-ppi")
    ip, ix = dev(indptr), dev(indices)
    w = weights_of(len(indices), "positive")
    with pytest.raises(TypeError):
        gs.WeightedNeighborSampler(ip, ix, dev(w.astype(np.float64)))
    with pytest.raises(ValueError):
        gs.WeightedNeighborSampler(ip, ix, dev(w[:-1]))
    with pytest.raises(ValueError):
        gs.WeightedNeighborSampler(ip, ix, torch.from_numpy(w))           # weights on the host
    tab = gs.ops.csr_alias_table(ip, ix, dev(w))
    with pytest.raises(RuntimeError):
        gs.ops.sample_alias(ip, tab, dev(np.zeros(4, np.int32)), 1025, 1, 0)
    with pytest.raises(RuntimeError):
        gs.ops.sample_alias_khop(ip, tab, dev(np.zeros(4, np.int32)), [65], 1, 0)
    with pytest.raises(RuntimeError):
        gs.ops.sample_alias_khop(ip, tab, dev(np.zeros(4, np.int32)), [2] * 5, 1, 0)
