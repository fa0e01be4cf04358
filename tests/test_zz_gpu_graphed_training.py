"""GPU: whole training steps captured in CUDA graphs (graphed_training.GraphedTrainStep).

Every replay is compared bit for bit (torch.equal) with an eager twin built with the same seeds and a capturable Adam:
the loss, every parameter and the RNG counters after each step.  Also: interleaved eager steps (the short last batch of
an epoch), the unsupervised three-pass step with shared negatives, Node2Vec, the device-side call offset of the three
dropout kernels, and the refusals."""
import numpy as np
import pytest
import torch

from conftest import load_golden
from oracle import dropout as od

pytestmark = pytest.mark.gpu

B, C = 24, 5


def _graph():
    g = load_golden("khop")
    return torch.from_numpy(g["adj"]).cuda(), torch.from_numpy(g["feats"]).cuda()


def _supervised(kind, sigmoid, d, rate, math, shared_sampler=True):
    import graphsage_b200 as gs
    adj, feats = _graph()
    gs.inits.manual_seed(11)
    gs.set_default_math(math)
    try:
        sampler = gs.UniformNeighborSampler(adj, seed=7)
        sampler.counter = 3
        other = sampler if shared_sampler else gs.UniformNeighborSampler(adj, seed=8)
        infos = [gs.SAGEInfo("node", sampler, 5, 16), gs.SAGEInfo("node", other, 3, 16)]
        m = gs.SupervisedGraphsage(C, {"batch_size": B, "dropout": rate}, feats, adj, None, infos, concat=kind != "gcn",
                                   aggregator_type=kind, sigmoid_loss=sigmoid, learning_rate=0.01, weight_decay=1e-3,
                                   identity_dim=d, dropout_seed=99)
    finally:
        gs.set_default_math("fp32")
    gen = torch.Generator(device="cuda").manual_seed(2)         # a non-zero MLP bias, the same for models built alike
    for a in m.aggregators:
        if hasattr(a, "mlp_layers"):
            bias = a.mlp_layers[0].vars["bias"]
            bias.data.add_(torch.randn(bias.shape, generator=gen, device=bias.device) * 0.1)
    return m


def _eager_twin(build, *args):
    import graphsage_b200 as gs
    m = build(*args)
    gs.make_adam_capturable(m.optimizer)
    return m


def _batches(n_steps, sigmoid, seed=5, sizes=None):
    rs = np.random.RandomState(seed)
    n = 300
    out = []
    for i in range(n_steps):
        b = B if sizes is None else sizes[i]
        ids = torch.from_numpy(rs.randint(0, n, size=b).astype(np.int32))
        if sigmoid:
            labels = (rs.rand(b, C) < 0.3).astype(np.float32)
        else:
            labels = np.eye(C, dtype=np.float32)[rs.randint(0, C, size=b)]
        out.append((ids, torch.from_numpy(labels)))
    return out


def _same_state(m, twin):
    assert all(torch.equal(p, q) for p, q in zip(m.parameters(), twin.parameters()))
    assert m.dropout_counter == twin.dropout_counter
    assert m.layer_infos[0].neigh_sampler.counter == twin.layer_infos[0].neigh_sampler.counter


@pytest.mark.parametrize("math", ["fp32", "tf32x3"])
@pytest.mark.parametrize("rate", [0.0, 0.5])
@pytest.mark.parametrize("sigmoid,d", [(True, 0), (False, 16), (True, 16), (False, 0)])
@pytest.mark.parametrize("kind", ["mean", "gcn", "maxpool", "meanpool"])
def test_supervised_replays_equal_eager_steps(kind, sigmoid, d, rate, math):
    args = (kind, sigmoid, d, rate, math)
    m, twin = _supervised(*args), _eager_twin(_supervised, *args)
    _same_state(m, twin)
    step = m.graphed_train_step(B)
    _same_state(m, twin)                                         # capturing the step neither trains nor draws
    for ids, labels in _batches(5, sigmoid):
        loss = step(ids.cuda(), labels.cuda())
        want = twin.train_step(ids, labels)
        assert torch.equal(loss, want), (float(loss), float(want))
        _same_state(m, twin)
    if rate:
        assert m.dropout_counter > 0


@pytest.mark.parametrize("kind,d,math", [("mean", 16, "fp32"), ("maxpool", 16, "tf32x3"), ("gcn", 0, "tf32x3")])
def test_graphed_eager_short_batch_graphed_equals_all_eager(kind, d, math):
    args = (kind, True, d, 0.5, math)
    m, twin = _supervised(*args), _eager_twin(_supervised, *args)
    step = m.graphed_train_step(B)
    data = _batches(5, True, seed=9, sizes=[B, B, B - 7, B, B])
    for i, (ids, labels) in enumerate(data):
        got = step(ids, labels) if ids.numel() == B else m.train_step(ids, labels)
        assert torch.equal(got, twin.train_step(ids, labels)), i
        _same_state(m, twin)
    # evaluation between replays sees the replayed weights: a replay changes them without a _version bump, so an eager
    # pack made before it must not be reused after it (no stale tensor-core weight images)
    for ids, labels in data[:2]:
        assert torch.equal(m.loss(ids, labels), twin.loss(ids, labels))
        assert torch.equal(step(ids, labels), twin.train_step(ids, labels))
        assert torch.equal(m.loss(ids, labels), twin.loss(ids, labels))
        assert torch.equal(m.predict(ids), twin.predict(ids))


def test_a_captured_step_repacks_weights_even_when_the_cache_key_matches():
    """Under capture every PackedWeights.get packs afresh inside the graph: a weight changed behind the cache's key (here
    through .data, which does not bump _version) is seen by the next replay."""
    import graphsage_b200 as gs
    from graphsage_b200 import ops
    dense = gs.Dense(40, 128, act=gs.identity, bias=False, math=ops.MATH_TF32X3)
    x = torch.randn(300, 40, device="cuda")
    dense(x)                                                     # eager: packs, the key now matches
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        g = torch.cuda.CUDAGraph()
        ops.REPACK_ALWAYS[0] = True
        try:
            g.capture_begin()
            y = dense(x)
            g.capture_end()
        finally:
            ops.REPACK_ALWAYS[0] = False
    torch.cuda.current_stream().wait_stream(s)
    W = dense.vars["weights"]
    W.data.mul_(-2.0)
    g.replay()
    want = ops.sage_gemm([(x, 40, W)], math=ops.MATH_TF32X3, packed=ops.PackedWeights())   # W packed as it is now
    assert not torch.equal(want, ops.sage_gemm([(x, 40, W * -0.5)], math=ops.MATH_TF32X3, packed=ops.PackedWeights()))
    assert torch.equal(y, want)


def _unsupervised(kind, rate):
    import graphsage_b200 as gs
    adj, feats = _graph()
    gs.inits.manual_seed(13)
    deg = np.random.RandomState(3).randint(1, 40, size=300).astype(np.float64)
    sampler = gs.UniformNeighborSampler(adj, seed=123)
    infos = [gs.SAGEInfo("node", sampler, 5, 12), gs.SAGEInfo("node", sampler, 3, 12)]
    return gs.UnsupervisedGraphsage({"batch_size": B, "dropout": rate}, feats, adj, deg, infos, concat=True,
                                    aggregator_type=kind, neg_sample_size=20, learning_rate=0.01, weight_decay=1e-3, seed=77,
                                    dropout_seed=31, identity_dim=8)


@pytest.mark.parametrize("rate", [0.0, 0.5])
@pytest.mark.parametrize("kind", ["mean", "maxpool"])
def test_unsupervised_three_passes_replay_equal_eager(kind, rate):
    m, twin = _unsupervised(kind, rate), _eager_twin(_unsupervised, kind, rate)
    step = m.graphed_train_step(B)
    rs = np.random.RandomState(4)
    for i in range(5):
        b1 = torch.from_numpy(rs.randint(0, 300, size=B).astype(np.int32))
        b2 = torch.from_numpy(rs.randint(0, 300, size=B).astype(np.int32))
        loss = step(b1, b2) if i != 3 else m.train_step(b1, b2)
        assert torch.equal(loss, twin.train_step(b1, b2)), i
        assert all(torch.equal(p, q) for p, q in zip(m.parameters(), twin.parameters()))
        assert m.neg_sampler.counter == twin.neg_sampler.counter == i + 1
        assert m.dropout_counter == twin.dropout_counter
        assert m.layer_infos[0].neigh_sampler.counter == twin.layer_infos[0].neigh_sampler.counter
    assert float(m.mrr()) == float(twin.mrr())


def _n2v():
    import graphsage_b200 as gs
    deg = np.random.RandomState(8).randint(1, 30, size=300)
    return gs.Node2VecModel(None, 301, deg, nodevec_dim=24, lr=0.05, neg_sample_size=20, seed=5)


def test_node2vec_replays_equal_eager():
    m, twin = _n2v(), _n2v()
    step = m.graphed_train_step(B)
    assert torch.equal(m._target, twin._target) and torch.equal(m._context, twin._context)
    rs = np.random.RandomState(6)
    for i in range(6):
        b = B if i != 2 else B - 5
        b1 = torch.from_numpy(rs.randint(0, 301, size=b).astype(np.int32)).cuda()
        b2 = torch.from_numpy(rs.randint(0, 301, size=b).astype(np.int32)).cuda()
        loss = step(b1, b2) if b == B else m.train_step(b1, b2)
        assert torch.equal(loss, twin.train_step(b1, b2)), i
        assert torch.equal(m.target_embeds, twin.target_embeds)
        assert torch.equal(m._context, twin._context)                # context rows and their biases
        assert m.neg_sampler.counter == twin.neg_sampler.counter == i + 1
    m.neg_sampler.check()
    twin.neg_sampler.check()


# ---------------------------------------------------------------------------------------------------- device call offset
def _dev(x):
    return torch.full((1,), x, dtype=torch.int64, device="cuda")


@pytest.mark.parametrize("c,x", [(9, 0), (9, 5), (2 ** 32 - 3, 7), (0, 2 ** 33 + 4)])
def test_dropout_apply_call_offset(c, x):
    import graphsage_b200 as gs
    rs = np.random.RandomState(1)
    xs = torch.from_numpy(rs.randn(130, 37).astype(np.float32)).cuda()
    got = gs.ops.dropout_apply(xs, (77, c, 0.4, _dev(x)))
    want = gs.ops.dropout_apply(xs, (77, (c + x) & 0xFFFFFFFF, 0.4))
    assert torch.equal(got, want)
    # call_dev NULL is the host-numbered site of the mask contract
    m = od.keep_mask(77, c, 0.4, np.arange(130), 37)
    ref = np.where(m, xs.cpu().numpy() / od.keep_prob(0.4), np.float32(0)).astype(np.float32)
    assert np.array_equal(gs.ops.dropout_apply(xs, (77, c, 0.4)).cpu().numpy(), ref)


@pytest.mark.parametrize("F,pitch", [(602, 608), (37, 37)])            # bulk-copy kernel, scalar fallback
def test_gather_mean_dropout_call_offset(F, pitch):
    import graphsage_b200 as gs
    rs = np.random.RandomState(F)
    N = 500
    table = torch.from_numpy(rs.randn(N, pitch).astype(np.float32)).cuda()[:, :F]
    s0 = torch.from_numpy(rs.randint(0, N, size=11).astype(np.int32)).cuda()
    s1 = torch.from_numpy(rs.randint(0, N, size=55).astype(np.int32)).cuda()
    s2 = torch.from_numpy(rs.randint(0, N, size=165).astype(np.int32)).cuda()
    segs = [gs.ops.Seg(11, 5, self_ids=s0, neigh_ids=s1, out_row0=0), gs.ops.Seg(55, 3, self_ids=s1, neigh_ids=s2, out_row0=11)]
    dn, ds = _dev(40), _dev(1000)                                   # different offsets for neighbour and self sites
    for include_self in (False, True):
        got = gs.ops.gather_mean_dropout(table, segs, [(5, 0, 0.5, dn), (5, 2, 0.3, dn)], [(5, 1, 0.5, ds), (5, 3, 0.3, ds)],
                                         include_self=include_self)
        want = gs.ops.gather_mean_dropout(table, segs, [(5, 40, 0.5), (5, 42, 0.3)], [(5, 1001, 0.5), (5, 1003, 0.3)],
                                          include_self=include_self)
        assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])
        zero = gs.ops.gather_mean_dropout(table, segs, [(5, 0, 0.5, _dev(0)), (5, 2, 0.3)], [(5, 1, 0.5), (5, 3, 0.3, _dev(0))],
                                          include_self=include_self)
        null = gs.ops.gather_mean_dropout(table, segs, [(5, 0, 0.5), (5, 2, 0.3)], [(5, 1, 0.5), (5, 3, 0.3)],
                                          include_self=include_self)
        assert torch.equal(zero[0], null[0]) and torch.equal(zero[1], null[1])


def test_embedding_grad_dropout_call_offset():
    import graphsage_b200 as gs
    rs = np.random.RandomState(2)
    n_rows, d = 400, 20
    ids1 = torch.from_numpy(rs.randint(0, n_rows, size=300).astype(np.int32)).cuda()
    ids2 = torch.from_numpy(rs.randint(0, 40, size=600).astype(np.int32)).cuda()      # long runs of repeated ids
    g1 = torch.from_numpy(rs.randn(300, d).astype(np.float32)).cuda()
    g2 = torch.from_numpy(rs.randn(200, d).astype(np.float32)).cuda()
    lists = [(ids1, g1, 1, 1.0), (ids2, g2, 3, 1.0 / 3)]
    got = gs.ops.embedding_grad(lists, n_rows, d, sites=[(9, 4, 0.5, _dev(6)), (9, 5, 0.2, _dev(2 ** 32 + 1))])
    want = gs.ops.embedding_grad(lists, n_rows, d, sites=[(9, 10, 0.5), (9, 6, 0.2)])
    assert torch.equal(got, want)
    null = gs.ops.embedding_grad(lists, n_rows, d, sites=[(9, 4, 0.5), (9, 5, 0.2)])
    assert torch.equal(gs.ops.embedding_grad(lists, n_rows, d, sites=[(9, 4, 0.5, _dev(0)), (9, 5, 0.2)]), null)


def test_replays_advanced_by_gs_bump_counter_draw_fresh_masks():
    """A graph bakes call = 3; gs_bump_counter inside the graph moves the device word, so replay r masks with call 3 + r."""
    import graphsage_b200 as gs
    x = torch.randn(64, 40, device="cuda")
    call_dev = _dev(0)
    out = torch.empty_like(x)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        gs.ops.dropout_apply(x, (1, 3, 0.5, call_dev), out=out)     # warm-up outside the graph
        g = torch.cuda.CUDAGraph()
        g.capture_begin()
        gs.ops.dropout_apply(x, (1, 3, 0.5, call_dev), out=out)
        gs.ops.check(gs.ops.lib().gs_bump_counter(call_dev.data_ptr(), 1, gs.ops.stream_ptr()))
        g.capture_end()
    torch.cuda.current_stream().wait_stream(s)
    for r in range(3):
        g.replay()
        assert torch.equal(out, gs.ops.dropout_apply(x, (1, 3 + r, 0.5))), r
    assert int(call_dev.item()) == 3


# ---------------------------------------------------------------------------------------------------- refusals
def test_refusals():
    m = _supervised("mean", True, 0, 0.5, "fp32")
    m.distributed = True
    with pytest.raises(NotImplementedError, match="distributed"):
        m.graphed_train_step(B)
    m2 = _supervised("mean", True, 0, 0.0, "fp32", shared_sampler=False)
    with pytest.raises(NotImplementedError, match="neigh_sampler"):
        m2.graphed_train_step(B)
    m3 = _supervised("maxpool", False, 0, 0.0, "fp32")
    step = m3.graphed_train_step(B)
    ids, labels = _batches(1, False)[0]
    with pytest.raises(ValueError, match="captured"):
        step(ids[:B - 1], labels[:B - 1])
    with pytest.raises(ValueError, match="captured"):
        step(ids, labels[:, :C - 1])
    u = _unsupervised("mean", 0.0).graphed_train_step(B)
    with pytest.raises(ValueError, match="captured"):
        u(ids, ids[:B - 2])
    n = _n2v().graphed_train_step(B)
    with pytest.raises(ValueError, match="captured"):
        n(torch.cat([ids, ids]), torch.cat([ids, ids]))
