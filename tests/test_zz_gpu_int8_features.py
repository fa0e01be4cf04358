"""GPU: int8 feature tables with a per-row scale (graphsage_b200.Int8Features, GS_I8ROW).

* gs_quantize_rows_i8 byte for byte against oracle/int8_rows.py.
* gs_gather_mean, gs_gather_rows_f32 and gs_sage_layer_small_i8 on int8 rows, bit for bit against the fp32 kernels on the
  dequantised table: ids and row ranges, include_self, want_self, out-of-range ids, several fanouts and widths.
* The model contract: every output, loss, gradient step and graph replay of a model over an Int8Features table is
  torch.equal to the same model over the fp32 table table.dequantize() - every aggregator that takes it, fp32 and tf32x3
  math, concat on and off, one layer of <= 2,048 rows (the one-launch layer) and two layers.
* HostFeatures over int8 rows: equal to the device int8 model, pitch bytes staged per row, no host synchronisation.
* The refusals."""
import numpy as np
import pytest
import torch

from oracle import int8_rows

pytestmark = pytest.mark.gpu

N, MD, B, NC = 300, 12, 24, 5


def _feats(n, F, seed=0):
    rs = np.random.RandomState(seed)
    x = (rs.randn(n + 1, F) * rs.choice([1e-3, 1.0, 50.0], size=(n + 1, 1))).astype(np.float32)
    x[rs.rand(n + 1) < 0.05] = 0                      # some all-zero rows besides the dummy
    x[n] = 0
    return x


# ------------------------------------------------------------------ kernels
@pytest.mark.parametrize("F", [1, 3, 4, 5, 37, 602, 1536])
def test_quantize_bytes_equal_the_oracle(F):
    import graphsage_b200 as gs
    x = _feats(257, F, seed=F)
    got = gs.ops.quantize_rows_i8(torch.from_numpy(x).cuda()).cpu().numpy()
    assert got.shape == (258, int8_rows.pitch(F)) and int8_rows.pitch(F) == gs._lib.lib().gs_i8row_pitch(F)
    assert np.array_equal(got, int8_rows.quantize_rows(x))
    t = gs.Int8Features(x)                            # a host table, quantised on the device in chunks
    assert np.array_equal(t.rows.numpy(), got) and not t.rows.is_cuda
    q, s = int8_rows.unpack(got, F)
    deq = int8_rows.dequantize(q, s)
    assert np.array_equal(t.dequantize().numpy(), deq)
    assert np.array_equal(gs.Int8Features(torch.from_numpy(x).cuda()).dequantize().cpu().numpy(), deq)


def test_chunked_quantisation_equals_one_launch(monkeypatch):
    import graphsage_b200 as gs
    from graphsage_b200 import int8_features
    x = _feats(1000, 37)
    whole = gs.Int8Features(x, device="cuda").rows.cpu()
    monkeypatch.setattr(int8_features, "QUANTIZE_CHUNK_BYTES", 37 * 4 * 77)
    assert torch.equal(gs.Int8Features(x).rows, whole)
    assert torch.equal(gs.Int8Features(x, device="cuda").rows.cpu(), whole)


def _seg_args(n_rows, n, k, seed, by_ids, oob):
    import graphsage_b200 as gs
    rs = np.random.RandomState(seed)
    if by_ids:
        lo, hi = (-3, n_rows + 3) if oob else (0, n_rows)
        self_ids = torch.from_numpy(rs.randint(lo, hi, size=n).astype(np.int32)).cuda()
        neigh_ids = torch.from_numpy(rs.randint(lo, hi, size=n * k).astype(np.int32)).cuda()
        return [gs.ops.Seg(n, k, self_ids=self_ids, neigh_ids=neigh_ids)]
    n = min(n, (n_rows - 1) // (k + 1))
    return [gs.ops.Seg(n, k, self_row0=0, neigh_row0=n)]


@pytest.mark.parametrize("F", [1, 5, 602, 1536])
@pytest.mark.parametrize("k", [1, 10, 25])
def test_gather_mean_equals_fp32_on_the_dequantised_table(F, k):
    import graphsage_b200 as gs
    t = gs.Int8Features(torch.from_numpy(_feats(400, F, seed=k)).cuda())
    deq = t.dequantize()
    for by_ids, oob in ((True, False), (True, True), (False, False)):
        for include_self in (False, True):
            for want_self in (False, True):
                segs = _seg_args(401, 97, k, F + k, by_ids, oob)
                a = gs.ops.gather_mean(t, segs, include_self=include_self, want_self=want_self)
                b = gs.ops.gather_mean(deq, segs, include_self=include_self, want_self=want_self)
                assert torch.equal(a[1], b[1]), (by_ids, oob, include_self)
                if want_self:
                    assert torch.equal(a[0], b[0])
    # several segments in one call (the layer-0 hops)
    segs = _seg_args(401, 40, k, 1, True, False) + [gs.ops.Seg(30, 3, self_ids=torch.arange(30, dtype=torch.int32).cuda(),
                                                               neigh_ids=torch.arange(90, dtype=torch.int32).cuda(),
                                                               out_row0=40)]
    assert torch.equal(gs.ops.gather_mean(t, segs)[1], gs.ops.gather_mean(deq, segs)[1])


def test_gather_mean_reddit_size():
    import graphsage_b200 as gs
    n, F, b = 20000, 602, 512
    rs = np.random.RandomState(0)
    t = gs.Int8Features(torch.from_numpy(_feats(n, F)).cuda())
    deq = t.dequantize()
    h1 = torch.from_numpy(rs.randint(0, n, size=b * 25).astype(np.int32)).cuda()
    h2 = torch.from_numpy(rs.randint(0, n, size=b * 250).astype(np.int32)).cuda()
    seeds = torch.from_numpy(rs.randint(0, n, size=b).astype(np.int32)).cuda()
    segs = [gs.ops.Seg(b, 25, self_ids=seeds, neigh_ids=h1), gs.ops.Seg(b * 25, 10, self_ids=h1, neigh_ids=h2, out_row0=b)]
    a, b_ = gs.ops.gather_mean(t, segs, want_self=True), gs.ops.gather_mean(deq, segs, want_self=True)
    assert torch.equal(a[0], b_[0]) and torch.equal(a[1], b_[1])


@pytest.mark.parametrize("F", [1, 5, 602])
def test_gather_rows_f32_equals_the_dequantised_rows(F):
    import graphsage_b200 as gs
    t = gs.Int8Features(torch.from_numpy(_feats(200, F)).cuda())
    deq = t.dequantize()
    ids = torch.tensor([0, 5, 199, 200, -1, 7000, 3], dtype=torch.int32).cuda()
    assert torch.equal(gs.ops.gather_rows_f32(t, ids), gs.ops.gather_rows_f32(deq, ids))
    assert torch.equal(gs.ops.gather_rows_f32(t, row0=150, n=51), gs.ops.gather_rows_f32(deq, row0=150, n=51))


@pytest.mark.parametrize("F,N_out,concat", [(5, 16, True), (37, 16, False), (64, 32, True), (602, 128, True)])
@pytest.mark.parametrize("include_self", [False, True])
def test_sage_layer_small_equals_fp32_on_the_dequantised_table(F, N_out, concat, include_self):
    import graphsage_b200 as gs
    t = gs.Int8Features(torch.from_numpy(_feats(300, F)).cuda())
    deq = t.dequantize()
    rs = np.random.RandomState(1)
    W = [torch.from_numpy(rs.randn(F, N_out).astype(np.float32)).cuda() for _ in range(2)]
    bias = torch.from_numpy(rs.randn(2 * N_out if concat else N_out).astype(np.float32)).cuda()
    parts = [(None, F, W[1])] if include_self else [(None, F, W[0]), (None, F, W[1])]
    combine = gs.ops.COMBINE_CONCAT if concat and not include_self else gs.ops.COMBINE_ADD
    if include_self:
        bias = bias[:N_out]
    for by_ids, oob in ((True, False), (True, True), (False, False)):
        seg = _seg_args(301, 45, 7, F, by_ids, oob)[0]
        kw = dict(combine=combine, include_self=include_self, bias=bias, act=gs.ops.ACT_RELU, l2_normalize=True)
        assert torch.equal(gs.ops.sage_layer_small(t, seg, parts, **kw), gs.ops.sage_layer_small(deq, seg, parts, **kw))


# ------------------------------------------------------------------ models against their dequantised twins
def _data(F=37, seed=0):
    rs = np.random.RandomState(seed)
    adj = rs.randint(0, N, size=(N + 1, MD)).astype(np.int32)
    adj[:N][rs.rand(N) < 0.1] = N
    adj[N] = N
    return adj, _feats(N, F, seed)


def _build(kind, features, adj, layers=2, cls="sage", math="fp32", concat=None, **kw):
    import graphsage_b200 as gs
    gs.inits.manual_seed(11)
    gs.set_default_math(math)
    try:
        adj_d = torch.from_numpy(adj).cuda()
        sampler = gs.UniformNeighborSampler(adj_d, seed=7)
        infos = [gs.SAGEInfo("node", sampler, f, 16) for f in [5, 3][:layers]]
        ph = {"batch_size": B, "dropout": kw.pop("dropout", 0.)}
        concat = kind != "gcn" if concat is None else concat
        if cls == "sage":
            return gs.SampleAndAggregate(ph, features, adj_d, None, infos, concat=concat, aggregator_type=kind)
        if cls == "sup":
            return gs.SupervisedGraphsage(NC, ph, features, adj_d, None, infos, concat=concat, aggregator_type=kind,
                                          learning_rate=0.01, weight_decay=1e-3, **kw)
        deg = np.random.RandomState(3).randint(1, 40, size=N).astype(np.float64)
        return gs.UnsupervisedGraphsage(ph, features, adj_d, deg, infos, concat=concat, aggregator_type=kind,
                                        neg_sample_size=7, learning_rate=0.01, weight_decay=1e-3, seed=77, **kw)
    finally:
        gs.set_default_math("fp32")


def _pair(kind, F=37, **kw):
    """(model on an Int8Features table, twin on its dequantised fp32 table), built alike."""
    import graphsage_b200 as gs
    adj, feats = _data(F)
    t = gs.Int8Features(torch.from_numpy(feats).cuda())
    return _build(kind, t, adj, **kw), _build(kind, t.dequantize(), adj, **kw)


def _first(fn, *a):
    import graphsage_b200 as gs
    gs.inits.manual_seed(12)
    return fn(*a)


def _ids(seed, b=B):
    return torch.from_numpy(np.random.RandomState(seed).randint(0, N, size=b).astype(np.int32))


def _labels(seed, sigmoid, b=B):
    rs = np.random.RandomState(seed + 100)
    lab = (rs.rand(b, NC) < 0.3) if sigmoid else np.eye(NC)[rs.randint(0, NC, size=b)]
    return torch.from_numpy(lab.astype(np.float32))


def _same_params(m, twin):
    return all(torch.equal(p, q) for p, q in zip(m.parameters(), twin.parameters()))


KINDS = ["mean", "gcn", "maxpool", "meanpool", "twomaxpool"]


@pytest.mark.parametrize("layers", [1, 2])
@pytest.mark.parametrize("math", ["fp32", "tf32x3"])
@pytest.mark.parametrize("kind,concat", [(k, c) for k in KINDS for c in (True, False) if not (k == "gcn" and c)])
def test_forward_equals_the_dequantised_twin(kind, concat, math, layers):
    """GCN combines one part, so its models are built with concat off (as the reference's graphsage_gcn)."""
    import graphsage_b200 as gs
    m, twin = _pair(kind, layers=layers, math=math, concat=concat)
    gs.set_default_math(math)
    try:
        assert torch.equal(_first(m.forward, _ids(0)), _first(twin.forward, _ids(0)))
        for s in range(1, 3):
            assert torch.equal(m.forward(_ids(s)), twin.forward(_ids(s))), s
    finally:
        gs.set_default_math("fp32")


def test_export_and_graphed_forward_equal_the_twin():
    m, twin = _pair("mean")
    ids = np.arange(0, N, 3)
    assert np.array_equal(_first(m.export_embeddings, ids, B), _first(twin.export_embeddings, ids, B))
    g = m.graphed(B)
    for s in range(3):
        assert torch.equal(g(_ids(s).cuda()).clone(), twin.forward(_ids(s))), s
    g.close()


@pytest.mark.parametrize("layers", [1, 2])
@pytest.mark.parametrize("math", ["fp32", "tf32x3"])
@pytest.mark.parametrize("kind", KINDS)
def test_supervised_training_equals_the_twin(kind, math, layers):
    m, twin = _pair(kind, cls="sup", math=math, layers=layers, sigmoid_loss=True)
    for s in range(5):
        ids, lab = _ids(s), _labels(s, True)
        assert torch.equal(m.train_step(ids, lab), twin.train_step(ids, lab)), s
        assert _same_params(m, twin), s
    assert torch.equal(m.predict(_ids(9)), twin.predict(_ids(9)))


@pytest.mark.parametrize("kind", ["mean", "maxpool"])
def test_unsupervised_training_equals_the_twin(kind):
    m, twin = _pair(kind, cls="unsup")
    for s in range(4):
        b1, b2 = _ids(s), _ids(s + 50)
        assert torch.equal(m.loss(b1, b2), twin.loss(b1, b2)), s
        assert torch.equal(m.train_step(b1, b2), twin.train_step(b1, b2)), s
        assert _same_params(m, twin), s


@pytest.mark.parametrize("cls,kind", [("sup", "mean"), ("sup", "maxpool"), ("unsup", "gcn")])
def test_graphed_train_step_replays_equal_the_twin(cls, kind):
    import graphsage_b200 as gs
    m, twin = _pair(kind, cls=cls)
    gs.make_adam_capturable(twin.optimizer)
    step = m.graphed_train_step(B)
    for s in range(4):
        a = (_ids(s), _labels(s, False)) if cls == "sup" else (_ids(s), _ids(s + 50))
        assert torch.equal(step(*[x.cuda() for x in a]), twin.train_step(*a)), s
        assert _same_params(m, twin), s


# ------------------------------------------------------------------ HostFeatures over int8 rows
@pytest.mark.parametrize("cached", [0.0, 0.3, 1.0])
@pytest.mark.parametrize("kind", ["mean", "maxpool"])
def test_host_int8_equals_the_device_int8_model(kind, cached):
    import graphsage_b200 as gs
    from graphsage_b200.host_features import hot_rows
    adj, feats = _data()
    dev = _build(kind, gs.Int8Features(torch.from_numpy(feats).cuda()), adj, cls="sup")
    hf = gs.HostFeatures(gs.Int8Features(feats), cache_ids=hot_rows(adj, int(cached * N)))
    host = _build(kind, hf, adj, cls="sup")
    assert hf.row_bytes == hf.pitch == int8_rows.pitch(feats.shape[1]) and hf.ws.dtype == torch.uint8
    assert hf.ws.shape[1] == int8_rows.pitch(feats.shape[1])
    assert torch.equal(_first(host.forward, _ids(0)), _first(dev.forward, _ids(0)))
    for s in range(4):
        ids, lab = _ids(s), _labels(s, False)
        assert torch.equal(host.train_step(ids, lab), dev.train_step(ids, lab)), s
        assert _same_params(host, dev), s
    hf.close()


def test_host_int8_step_does_not_synchronise():
    import graphsage_b200 as gs
    from graphsage_b200.host_features import hot_rows
    adj, feats = _data()
    hf = gs.HostFeatures(gs.Int8Features(feats), cache_ids=hot_rows(adj, N // 3))
    m = _build("mean", hf, adj, cls="sup")
    ids, lab = _ids(0).cuda(), _labels(0, False).cuda()
    m.train_step(ids, lab)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        m.train_step(ids, lab)
        m.forward(ids)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    hf.close()


# ------------------------------------------------------------------ refusals
def test_refusals():
    import graphsage_b200 as gs
    adj, feats = _data()
    t = gs.Int8Features(torch.from_numpy(feats).cuda())
    hf = gs.HostFeatures(gs.Int8Features(feats))
    for table in (t, hf):
        with pytest.raises(NotImplementedError, match="fused_pool=True with an int8"):
            _build("maxpool", table, adj, cls="sup", fused_pool=True)
        with pytest.raises(NotImplementedError, match="seq aggregator with a torch.int8 feature table"):
            _build("seq", table, adj, cls="sup")
        with pytest.raises(NotImplementedError, match="training dropout with a torch.int8 feature table"):
            _build("mean", table, adj, cls="unsup", dropout=0.5)
    with pytest.raises(NotImplementedError, match="identity_dim > 0 with an int8"):
        gs.SampleAndAggregate({}, t, torch.from_numpy(adj).cuda(), None, [], identity_dim=4)
    with pytest.raises(NotImplementedError, match="distributed=True with an int8"):
        gs.SupervisedGraphsage(3, {}, t, None, np.ones(N), [], distributed=True)
    m = _build("mean", t, adj, cls="sup")
    indptr = torch.arange(N + 1, dtype=torch.int64)
    indices = torch.zeros(N, dtype=torch.int32)
    for call in (lambda: m.full_neighbor_embeddings(indptr, indices),
                 lambda: m.full_neighbor_minibatch_embeddings(indptr, indices, [0, 1]),
                 lambda: m.full_neighbor_train_step(indptr, indices, [0, 1], torch.zeros((2, NC))),
                 lambda: m.full_neighbor_minibatch_train_step(indptr, indices, [0, 1], torch.zeros((2, NC))),
                 lambda: m.full_neighbor_predict(indptr, indices, [0, 1])):
        with pytest.raises(NotImplementedError, match="full-neighbourhood .* with an int8"):
            call()
    with pytest.raises(ValueError, match="HostFeatures"):
        _build("mean", gs.Int8Features(feats), adj)
    hf.close()
