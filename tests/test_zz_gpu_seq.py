"""GPU: the LSTM sequence aggregator (graphsage_seq).  gs_seq_lengths bit for bit against the oracle's length rule;
gs_lstm_forward / gs_lstm_backward against the fp64 oracle fed the same P and dh_last; the aggregator and the model
against the oracle (forward, graphed, the dense call path; fp32 and tf32x3); the supervised and unsupervised training
steps against torch-CPU autograd on the oracle's op sequence; determinism; graph replays equal to eager steps; toy-ppi
training; peak memory; the refusals."""
import numpy as np
import pytest
import torch

from conftest import load_golden, rel_err
from oracle import seq as oseq

pytestmark = pytest.mark.gpu

TOL = 1e-4


def test_seq_lengths_bit_for_bit():
    import graphsage_b200 as gs
    rs = np.random.RandomState(1)
    n, k, K = 301, 7, 37
    x = rs.randn(n, k, K).astype(np.float32)
    x[rs.rand(n, k) < 0.3] = 0.0                    # interspersed zero rows
    x[5] = 0.0                                      # an all-zero sequence: len 1
    x[6, :4] = -0.0                                 # negative zeros are zero
    x[7] = 0.0
    x[7, :, -1] = 1.0                               # one non-zero element per row, in the last column
    buf = torch.zeros((n * k, 40), device="cuda")   # strided rows (ld 40 > K)
    buf[:, :K] = torch.from_numpy(x.reshape(n * k, K)).cuda()
    got = gs.ops.seq_lengths(buf[:, :K], n, k).cpu().numpy()
    assert np.array_equal(got, oseq.seq_lengths(x))
    assert got[5] == 1 and got[7] == k


@pytest.mark.parametrize("k", [1, 10, 25])
@pytest.mark.parametrize("H", [128, 256])
def test_lstm_kernels_against_fp64_oracle(H, k):
    import graphsage_b200 as gs
    rs = np.random.RandomState(H + k)
    n, K = 45, 20                                    # not a multiple of the 32- / 16-sequence tile
    r = np.sqrt(6.0 / (K + 5 * H))
    kernel = rs.uniform(-r, r, size=(K + H, 4 * H)).astype(np.float32)
    P = (rs.randn(n * k, 4 * H) * 0.8).astype(np.float32)
    lengths = rs.randint(1, k + 1, size=n).astype(np.int32)
    lengths[:3] = [1, k, max(1, k // 2)]
    kt = torch.from_numpy(kernel).cuda()
    h, g, c, hp = gs.ops.lstm_forward(torch.from_numpy(P).cuda(), kt[K:], torch.from_numpy(lengths).cuda(), n, k, train=True)
    h_only = gs.ops.lstm_forward(torch.from_numpy(P).cuda(), kt[K:], torch.from_numpy(lengths).cuda(), n, k)
    assert torch.equal(h, h_only)
    rh, rg, rc, rhp = oseq.lstm_run(P.reshape(n, k, 4 * H), kernel[K:], lengths, train=True, dtype=np.float64)
    errs = {"h_last": np.abs(h.cpu().numpy() - rh).max(), "gates": np.abs(g.cpu().numpy() - rg.reshape(n * k, -1)).max(),
            "c": np.abs(c.cpu().numpy() - rc.reshape(n * k, -1)).max(), "h_prev": np.abs(hp.cpu().numpy() - rhp.reshape(n * k, -1)).max()}
    dh = rs.randn(n, H).astype(np.float32)
    dZ = gs.ops.lstm_backward(torch.from_numpy(dh).cuda(), g, c, torch.from_numpy(lengths).cuda(), kt[K:], n, k)
    rdZ = oseq.lstm_bptt(dh, rg, rc, lengths, kernel[K:]).reshape(n * k, -1)
    errs["dZ"] = np.abs(dZ.cpu().numpy() - rdZ).max()
    print("H=%d k=%d max abs errors: %s" % (H, k, {a: "%.2e" % b for a, b in errs.items()}))
    assert max(errs["h_last"], errs["gates"], errs["c"], errs["h_prev"]) < 1e-5, errs
    assert errs["dZ"] < 2e-5, errs
    past = np.arange(k)[None, :] >= lengths[:, None]
    assert not g.cpu().numpy().reshape(n, k, -1)[past].any() and not dZ.cpu().numpy().reshape(n, k, -1)[past].any()


def _model(math, concat=True, dropout=0.0, size="small", B=16, fan=(5, 3), cls=None, **kw):
    import graphsage_b200 as gs
    g = load_golden("khop")
    gs.inits.manual_seed(11)
    gs.set_default_math(math)
    try:
        sampler = gs.UniformNeighborSampler(torch.from_numpy(g["adj"]).cuda(), seed=123)
        sampler.counter = 40
        infos = [gs.SAGEInfo("node", sampler, fan[0], 12), gs.SAGEInfo("node", sampler, fan[1], 8)]
        args = ({"batch_size": B, "dropout": dropout}, torch.from_numpy(g["feats"]).cuda(), torch.from_numpy(g["adj"]).cuda())
        if cls is None:
            m = gs.SampleAndAggregate(*args, None, infos, concat=concat, aggregator_type="seq", model_size=size, **kw)
        else:
            m = cls(*args, None, infos, concat=concat, aggregator_type="seq", model_size=size, **kw)
    finally:
        gs.set_default_math("fp32")
    gen = torch.Generator(device="cuda").manual_seed(2)
    return m, g, gen


def _oracle_aggs(aggs, dtype=np.float64):
    return [dict(kernel=a.cell.vars["kernel"].detach().cpu().numpy().astype(dtype),
                 cell_bias=a.cell.vars["bias"].detach().cpu().numpy().astype(dtype),
                 neigh_weights=a.vars["neigh_weights"].detach().cpu().numpy().astype(dtype),
                 self_weights=a.vars["self_weights"].detach().cpu().numpy().astype(dtype)) for a in aggs]


@pytest.mark.parametrize("math", ["fp32", "tf32x3"])
@pytest.mark.parametrize("concat,size", [(True, "small"), (False, "big")])
def test_model_forward_graphed_and_dense_call_match_oracle(math, concat, size):
    import graphsage_b200 as gs
    import oracle
    outs = {}
    for rate in (0.0, 0.5):
        m, g, gen = _model(math, concat, rate, size)
        m.forward(torch.zeros(16, dtype=torch.int32))            # creates the aggregators (dropout = rate, never applied)
        for a in m.aggregators:
            a.cell.vars["bias"].add_(torch.randn(a.cell.vars["bias"].shape, generator=gen, device="cuda") * 0.2)
        seeds = np.random.RandomState(4).randint(0, 300, size=16).astype(np.int32)
        seeds[0] = 3                                             # node 3's neighbours are all the dummy id: len 1
        sampler = m.layer_infos[0].neigh_sampler
        c0 = sampler.counter
        out = m.forward(torch.from_numpy(seeds), normalize=False).cpu().numpy()
        samples, support = oracle.sample_khop(g["adj"], seeds, [5, 3], 123, c0)
        ref = oseq.aggregate_khop_seq(samples, g["feats"], [5, 3], support, 16, _oracle_aggs(m.aggregators), concat,
                                      dtype=np.float64)
        assert rel_err(out, ref) < TOL, (math, rel_err(out, ref))
        sampler.counter = c0
        run = m.graphed(16, normalize=False)
        got = run(torch.from_numpy(seeds).cuda()).cpu().numpy()
        run.close()
        assert np.array_equal(got, out)
        # the dense call path: the reference's agg((self_vecs, neigh_vecs)) on materialised rows, layer 0 hop 0
        a0 = m.aggregators[0]
        dense = a0((torch.from_numpy(g["feats"][samples[0]]).cuda(), torch.from_numpy(g["feats"][samples[1]]).cuda().reshape(16, 3, -1)))
        w = _oracle_aggs([a0])[0]
        want = oseq.seq_aggregator(g["feats"][samples[0]], g["feats"][samples[1]].reshape(16, 3, -1), w["kernel"], w["cell_bias"],
                                   w["neigh_weights"], w["self_weights"], concat, dtype=np.float64)
        assert rel_err(dense.cpu().numpy(), want) < TOL
        outs[rate] = out
    assert np.array_equal(outs[0.0], outs[0.5])                  # the rate changes nothing: no aggregator dropout


def _cpu_logits_out(g, seeds, samples_fn, aggs, concat, emb=None):
    feats = torch.from_numpy(g["feats"]).double()
    table = torch.cat([emb, feats], dim=1) if emb is not None else feats
    samples, support = samples_fn(seeds)
    hidden = [table.index_select(0, torch.from_numpy(np.asarray(s)).long()) for s in samples]
    fan = [5, 3]
    for layer in range(2):
        a, nxt = aggs[layer], []
        for hop in range(2 - layer):
            k = fan[1 - hop]
            nxt.append(oseq.torch_seq_layer(hidden[hop], hidden[hop + 1], a["kernel"], a["cell_bias"], a["self_weights"],
                                            a["neigh_weights"], k, concat, layer == 1))
        hidden = nxt
    out = hidden[0]
    return out / torch.sqrt(torch.clamp((out * out).sum(dim=1, keepdim=True), min=1e-12))


def _torch_aggs(m):
    return [{k: v.detach().cpu().double().clone().requires_grad_(True) for k, v in
             dict(kernel=a.cell.vars["kernel"], cell_bias=a.cell.vars["bias"], **a.vars).items()} for a in m.aggregators]


@pytest.mark.parametrize("concat,d,rate", [(True, 0, 0.0), (False, 0, 0.0), (True, 16, 0.0), (True, 0, 0.5),
                                           (False, 16, 0.5)])
def test_supervised_loss_gradients_and_adam_track_cpu(concat, d, rate):
    import graphsage_b200 as gs
    import oracle
    Cn, wd = 5, 1e-3
    m, g, gen = _model("fp32", concat, rate, cls=lambda *a, **k: gs.SupervisedGraphsage(Cn, *a, **k), sigmoid_loss=True,
                       learning_rate=0.01, weight_decay=wd, identity_dim=d, dropout_seed=7)
    for a in m.aggregators:
        a.cell.vars["bias"].data.add_(torch.randn(a.cell.vars["bias"].shape, generator=gen, device="cuda") * 0.2)
    aggs = _torch_aggs(m)
    head = {k: v.detach().cpu().double().clone().requires_grad_(True) for k, v in m.node_pred_vars.items()}
    emb = m.embeds.detach().cpu().double().clone().requires_grad_(True) if d else None
    cpu_params = [a[k] for a in aggs for k in ("neigh_weights", "self_weights")] + \
        [a[k] for a in aggs for k in ("kernel", "cell_bias")] + list(head.values()) + ([emb] if d else [])
    opt = torch.optim.Adam(cpu_params, lr=0.01)
    rs = np.random.RandomState(6)
    sampler = m.layer_infos[0].neigh_sampler
    for step in range(5):
        seeds = rs.randint(0, 300, size=16).astype(np.int32)
        labels = (rs.rand(16, Cn) < 0.3).astype(np.float32)
        c0, call0 = sampler.counter, m.dropout_counter
        out = _cpu_logits_out(g, seeds, lambda s: oracle.sample_khop(g["adj"], s, [5, 3], 123, c0), aggs, concat, emb)
        if rate:                                                  # the head's mask, read back from the kernel that draws it
            site = (m.dropout_key, call0, rate, None)
            out = out * gs.ops.dropout_apply(torch.ones(out.shape, device="cuda"), site).cpu().double()
        ref = torch.nn.functional.binary_cross_entropy_with_logits(out @ head["weights"] + head["bias"],
                                                                   torch.from_numpy(labels).double())
        for t in [a["neigh_weights"] for a in aggs] + [a["self_weights"] for a in aggs] + list(head.values()):
            ref = ref + wd * 0.5 * (t * t).sum()                  # the cell's kernel and bias are not decayed
        opt.zero_grad()
        ref.backward()
        if step == 0:                                             # the gradients of the first step, before any update
            m.optimizer.zero_grad(set_to_none=True)
            loss = m.loss(torch.from_numpy(seeds), torch.from_numpy(labels), dropout=rate)
            loss.backward()
            assert abs(float(loss) - float(ref)) < 2e-4 * max(1.0, abs(float(ref)))
            for p, q in zip(m.parameters(), cpu_params):
                assert rel_err(p.grad.cpu().numpy().reshape(1, -1), q.grad.numpy().reshape(1, -1), floor=1e-8) < 2e-4
            sampler.counter, m.dropout_counter = c0, call0
        for q in cpu_params:
            q.grad.clamp_(-5.0, 5.0)
        opt.step()
        m.train_step(torch.from_numpy(seeds), torch.from_numpy(labels))
        assert m.dropout_counter == call0 + (1 if rate else 0)    # the head site only
    for p, q in zip(m.parameters(), cpu_params):
        assert rel_err(p.detach().cpu().numpy().reshape(1, -1), q.detach().numpy().reshape(1, -1)) < 2e-4


def test_unsupervised_loss_and_gradients_match_cpu_autograd():
    import graphsage_b200 as gs
    import oracle
    deg = np.random.RandomState(3).randint(1, 40, size=301).astype(np.float64)
    m, g, gen = _model("fp32", True, 0.0, cls=lambda *a, **k: gs.UnsupervisedGraphsage(a[0], a[1], a[2], deg, a[4], **k),
                       neg_sample_size=7, learning_rate=0.01, seed=77)
    aggs = _torch_aggs(m)
    rs = np.random.RandomState(2)
    b1, b2 = rs.randint(0, 300, size=16).astype(np.int32), rs.randint(0, 300, size=16).astype(np.int32)
    sampler = m.layer_infos[0].neigh_sampler
    c0, n0 = sampler.counter, m.neg_sampler.counter
    loss = m.loss(torch.from_numpy(b1), torch.from_numpy(b2))
    loss.backward()
    m.neg_sampler.counter = n0
    neg = m.neg_sampler(7).cpu().numpy().astype(np.int32)
    outs = [_cpu_logits_out(g, s, lambda x, c=c: oracle.sample_khop(g["adj"], x, [5, 3], 123, c), aggs, True)
            for s, c in ((b1, c0), (b2, c0 + 2), (neg, c0 + 4))]
    o1, o2, on = outs
    aff = (o1 * o2).sum(dim=1)                                    # prediction.py:68-110, bilinear_weights=False
    neg_aff = o1 @ on.t()
    ref = (torch.nn.functional.binary_cross_entropy_with_logits(aff, torch.ones_like(aff), reduction="sum")
           + torch.nn.functional.binary_cross_entropy_with_logits(neg_aff, torch.zeros_like(neg_aff), reduction="sum")) / 16
    ref.backward()
    assert abs(float(loss) - float(ref)) < 2e-4 * max(1.0, abs(float(ref)))
    for p, q in zip(m.parameters(), [t for a in aggs for t in (a["neigh_weights"], a["self_weights"])] +
                    [t for a in aggs for t in (a["kernel"], a["cell_bias"])]):
        assert rel_err(p.grad.cpu().numpy().reshape(1, -1), q.grad.numpy().reshape(1, -1), floor=1e-8) < 2e-4


def test_training_is_deterministic():
    import graphsage_b200 as gs
    states = []
    for _ in range(2):
        m, g, gen = _model("tf32x3", True, 0.5, cls=lambda *a, **k: gs.SupervisedGraphsage(5, *a, **k), sigmoid_loss=True,
                           identity_dim=16)
        rs = np.random.RandomState(8)
        for _ in range(3):
            m.train_step(torch.from_numpy(rs.randint(0, 300, size=16).astype(np.int32)),
                         torch.from_numpy((rs.rand(16, 5) < 0.3).astype(np.float32)))
        states.append([p.detach().clone() for p in m.parameters()])
    assert all(torch.equal(a, b) for a, b in zip(*states))


@pytest.mark.parametrize("math,d", [("fp32", 0), ("tf32x3", 16)])
def test_graphed_train_step_equals_eager_twin(math, d):
    import graphsage_b200 as gs

    def build():
        m, _, gen = _model(math, True, 0.5, cls=lambda *a, **k: gs.SupervisedGraphsage(5, *a, **k), sigmoid_loss=True,
                           identity_dim=d, weight_decay=1e-3, dropout_seed=99)
        return m
    m, twin = build(), build()
    gs.make_adam_capturable(twin.optimizer)
    step = m.graphed_train_step(16)
    rs = np.random.RandomState(9)
    for i, b in enumerate([16, 16, 9, 16, 16]):
        ids = torch.from_numpy(rs.randint(0, 300, size=b).astype(np.int32))
        labels = torch.from_numpy((rs.rand(b, 5) < 0.3).astype(np.float32))
        got = step(ids, labels) if b == 16 else m.train_step(ids, labels)
        assert torch.equal(got, twin.train_step(ids, labels)), i
        assert all(torch.equal(p, q) for p, q in zip(m.parameters(), twin.parameters())), i
        assert m.dropout_counter == twin.dropout_counter


def test_toy_ppi_training_lowers_the_loss_and_peak_memory():
    import graphsage_b200 as gs
    g = load_golden("toy_ppi")
    n = g["feats"].shape[0]
    src = np.concatenate([g["src"], g["dst"]]).astype(np.int64)
    dst = np.concatenate([g["dst"], g["src"]]).astype(np.int64)
    order = np.argsort(src, kind="stable")
    indptr = np.zeros(n + 1, np.int64)
    np.cumsum(np.bincount(src, minlength=n), out=indptr[1:])
    adj, _ = gs.ops.build_padded_adj(torch.from_numpy(indptr).cuda(), torch.from_numpy(dst[order].astype(np.int32)).cuda(), 32)
    feats = torch.zeros((n + 1, 50), dtype=torch.float32, device="cuda")
    feats[:n] = torch.from_numpy(np.asarray(g["feats"], np.float32)).cuda()
    labels_all = (np.asarray(g["labels"]) > 0).astype(np.float32)
    gs.inits.manual_seed(3)
    sampler = gs.UniformNeighborSampler(adj, seed=1)
    infos = [gs.SAGEInfo("node", sampler, 10, 64), gs.SAGEInfo("node", sampler, 5, 64)]
    m = gs.SupervisedGraphsage(labels_all.shape[1], {"batch_size": 64, "dropout": 0.}, feats, adj, None, infos,
                               aggregator_type="seq", sigmoid_loss=True, learning_rate=0.01)
    rs = np.random.RandomState(0)
    losses = []
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    for i in range(50):
        if i == 1:                                   # Adam's state exists after the first step
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            base = torch.cuda.memory_allocated()
        ids = rs.randint(0, n, size=64).astype(np.int32)
        losses.append(float(m.train_step(torch.from_numpy(ids), torch.from_numpy(labels_all[ids]))))
    peak = torch.cuda.max_memory_allocated() - base
    print("seq toy-ppi: loss %.4f -> %.4f (mean of the last 5), peak above resident %.1f MB"
          % (losses[0], np.mean(losses[-5:]), peak / 2**20))
    assert np.mean(losses[-5:]) < 0.9 * losses[0]
    assert peak < 128 * 2**20


def test_refusals():
    import graphsage_b200 as gs
    g = load_golden("khop")
    adj = torch.from_numpy(g["adj"]).cuda()
    sampler = gs.UniformNeighborSampler(adj, seed=1)
    infos = [gs.SAGEInfo("node", sampler, 5, 8), gs.SAGEInfo("node", sampler, 3, 8)]
    bf = torch.from_numpy(g["feats"]).cuda().to(torch.bfloat16)
    with pytest.raises(NotImplementedError, match="bfloat16"):
        gs.SupervisedGraphsage(3, {"batch_size": 8}, bf, adj, None, infos, aggregator_type="seq")
    with pytest.raises(NotImplementedError, match="fused_pool"):
        gs.SupervisedGraphsage(3, {"batch_size": 8}, torch.from_numpy(g["feats"]).cuda(), adj, None, infos,
                               aggregator_type="seq", fused_pool=True)
    with pytest.raises(RuntimeError, match="H must be 128 or 256"):
        gs.ops.lstm_forward(torch.zeros((4, 256), device="cuda"), torch.zeros((64, 256), device="cuda"),
                            torch.ones(4, dtype=torch.int32, device="cuda"), 4, 1)
