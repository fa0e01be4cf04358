"""GPU: a feature table in host memory (graphsage_b200.HostFeatures).

* The staging passes (claim, gs_host_fetch, gs_host_translate) against oracle/host_stage.py, fp32 and bf16, F = 37 and
  602: the staged count, the staged rows byte for byte against the host rows, and the rows the translated ids address.
* Every output, loss and parameter of a model on a HostFeatures table is torch.equal to its twin on the same table held
  on the device: forward for every aggregator, the fused bf16 pooling kernel, 2 and 3 layers, no / the 30 % hottest / all
  rows cached, export_embeddings; supervised and unsupervised training, dropout, fused_pool training over several steps.
* CUDA-graph replays of the forward and of the training step; no host synchronisation in a step; the device memory a
  host table adds; the refusals."""
import numpy as np
import pytest
import torch

from oracle import host_stage

pytestmark = pytest.mark.gpu

N, MD, B, NC = 300, 12, 24, 5


def _data(F=37, seed=0):
    rs = np.random.RandomState(seed)
    adj = rs.randint(0, N, size=(N + 1, MD)).astype(np.int32)
    adj[:N][rs.rand(N) < 0.1] = N                 # nodes without neighbours sample the dummy id
    adj[N] = N
    feats = rs.randn(N + 1, F).astype(np.float32)
    feats[N] = 0
    return adj, feats


def _cache(adj, which):
    from graphsage_b200.host_features import hot_rows
    return {"none": None, "hot": hot_rows(adj, int(0.3 * N)), "all": np.arange(N)}[which]


def _bits(t):
    return t.view(torch.int16) if t.dtype == torch.bfloat16 else t.view(torch.int32)


# ------------------------------------------------------------------ the staging passes
@pytest.mark.parametrize("cache", ["none", "some", "all"])
@pytest.mark.parametrize("F", [37, 602])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_staging_against_the_oracle(dtype, F, cache):
    import graphsage_b200 as gs
    n = 500
    rs = np.random.RandomState(F)
    table = rs.randn(n + 1, F).astype(np.float32)
    table[n] = 0
    host = torch.from_numpy(table).to(dtype)
    cache_ids = {"none": np.zeros(0, np.int64), "some": np.array([3, 100, 250, 499]), "all": np.arange(n)}[cache]
    lists = [np.array([5, 5, 17, n, -1, 3, n + 7, 100, 5]),                          # repeats, dummy, out of range, hits
             np.zeros(0, np.int64),                                                    # an empty list
             np.array([17, 3, 250, 250, 2 ** 31 - 1, 499, 0]),                        # ids shared with the first list
             rs.randint(-5, n + 5, size=2000)]
    hf = gs.HostFeatures(host, cache_ids=cache_ids)
    try:
        ws, tr = hf.stage([torch.from_numpy(x.astype(np.int32)).cuda() for x in lists])
        ref_ws, ref_tr, staged = host_stage.stage(host.float().numpy(), lists, cache_ids)
        count, C = int(hf.count), len(cache_ids)
        assert count == len(staged)
        assert ws.shape[1] == F and ws.stride(0) == gs.ops.pad_cols(F)
        full = hf.ws                                                                   # the whole pitch, pad included
        padded = torch.zeros((n + 1, gs.ops.pad_cols(F)), dtype=dtype)
        padded[:, :F] = host
        # every staged id owns exactly one slot in [0, count) and its staged row is the host row, byte for byte
        slot, cached = {}, set(cache_ids.tolist())
        for ids, rows in zip(lists, tr):
            rows = rows.cpu().numpy()
            assert rows.shape == ids.shape and (rows >= 0).all()
            for i, r in zip(ids.tolist(), rows.tolist()):
                if 0 <= i < n and i not in cached:
                    assert C + 1 <= r < C + 1 + count
                    assert slot.setdefault(i, r) == r
        assert sorted(slot) == sorted(staged.tolist()) and sorted(slot.values()) == list(range(C + 1, C + 1 + count))
        got_rows = full[torch.tensor(list(slot.values()), dtype=torch.long)].cpu()
        assert torch.equal(_bits(got_rows), _bits(padded[torch.tensor(list(slot), dtype=torch.long)]))
        assert torch.equal(_bits(full[:C].cpu()), _bits(padded[torch.from_numpy(cache_ids)]))
        assert not _bits(full[C].cpu()).any()
        # the rows each translated id addresses are the oracle's, i.e. table[clamp(id)]
        for ids, rows, ref in zip(lists, tr, ref_tr):
            got = ws[rows.long()].cpu()
            assert torch.equal(_bits(got), _bits(torch.from_numpy(ref_ws[ref]).to(dtype)))
            assert torch.equal(_bits(got), _bits(host[torch.from_numpy(host_stage.clamp_ids(ids, n))]))
    finally:
        hf.close()


# ------------------------------------------------------------------ models against their device-table twins
def _build(kind, features, adj, layers=2, cls="sage", math="fp32", **kw):
    import graphsage_b200 as gs
    gs.inits.manual_seed(11)
    gs.set_default_math(math)
    try:
        adj_d = torch.from_numpy(adj).cuda()
        sampler = gs.UniformNeighborSampler(adj_d, seed=7)
        infos = [gs.SAGEInfo("node", sampler, f, 16) for f in [5, 3, 2][:layers]]
        ph = {"batch_size": B, "dropout": kw.pop("dropout", 0.)}
        concat = kind != "gcn"
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


def _pair(kind, cache="hot", dtype=torch.float32, F=37, **kw):
    """(model on a HostFeatures table, twin on the same table in HBM), built alike."""
    import graphsage_b200 as gs
    adj, feats = _data(F)
    t = torch.from_numpy(feats).to(dtype)
    hf = gs.HostFeatures(t, cache_ids=_cache(adj, cache))
    return _build(kind, hf, adj, **kw), _build(kind, t.cuda(), adj, **kw), hf


def _first(fn, *a):
    """fn(*a) with the weight initialiser reseeded: SampleAndAggregate creates its aggregators on the first forward."""
    import graphsage_b200 as gs
    gs.inits.manual_seed(12)
    return fn(*a)


def _ids(seed, b=B):
    return torch.from_numpy(np.random.RandomState(seed).randint(0, N, size=b).astype(np.int32))


def _labels(seed, sigmoid, b=B):
    rs = np.random.RandomState(seed + 100)
    lab = (rs.rand(b, NC) < 0.3) if sigmoid else np.eye(NC)[rs.randint(0, NC, size=b)]
    return torch.from_numpy(lab.astype(np.float32))


@pytest.mark.parametrize("cache", ["none", "hot", "all"])
@pytest.mark.parametrize("layers", [2, 3])
@pytest.mark.parametrize("kind", ["mean", "gcn", "maxpool", "meanpool", "twomaxpool", "seq"])
def test_forward_equals_the_device_table(kind, layers, cache):
    m, twin, hf = _pair(kind, cache, layers=layers)
    assert torch.equal(_first(m.forward, _ids(0)), _first(twin.forward, _ids(0)))
    for s in range(1, 3):
        assert torch.equal(m.forward(_ids(s)), twin.forward(_ids(s))), s


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("kind", ["maxpool", "meanpool"])
def test_fused_pool_forward_equals_the_device_table(kind, dtype):
    import graphsage_b200 as gs
    m, twin, hf = _pair(kind, "hot", dtype=dtype, math="bf16")
    gs.set_default_math("bf16")                         # the aggregators are created (with bf16 math) on the first forward
    try:
        assert torch.equal(_first(m.forward, _ids(0)), _first(twin.forward, _ids(0)))
        for s in range(1, 3):                           # several steps: a stale bf16 cast would show from the second on
            assert torch.equal(m.forward(_ids(s)), twin.forward(_ids(s))), s
    finally:
        gs.set_default_math("fp32")


def test_export_embeddings_equal_the_device_table():
    m, twin, hf = _pair("mean", "hot")
    ids = np.arange(0, N, 3)
    assert np.array_equal(_first(m.export_embeddings, ids, B), _first(twin.export_embeddings, ids, B))


def _same_params(m, twin):
    return all(torch.equal(p, q) for p, q in zip(m.parameters(), twin.parameters()))


@pytest.mark.parametrize("kind,sigmoid,cache", [("mean", False, "hot"), ("mean", True, "none"), ("gcn", True, "all"),
                                                ("maxpool", False, "hot"), ("seq", True, "hot")])
def test_supervised_training_equals_the_device_table(kind, sigmoid, cache):
    m, twin, hf = _pair(kind, cache, cls="sup", sigmoid_loss=sigmoid)
    for s in range(5):
        ids, lab = _ids(s), _labels(s, sigmoid)
        assert torch.equal(m.train_step(ids, lab), twin.train_step(ids, lab)), s
        assert _same_params(m, twin), s
    assert torch.equal(m.predict(_ids(9)), twin.predict(_ids(9)))


def test_supervised_dropout_training_equals_the_device_table():
    m, twin, hf = _pair("mean", "hot", cls="sup", dropout=0.5)
    for s in range(5):
        ids, lab = _ids(s), _labels(s, False)
        assert torch.equal(m.train_step(ids, lab), twin.train_step(ids, lab)), s
        assert _same_params(m, twin), s
    assert m.dropout_counter == twin.dropout_counter > 0


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_fused_pool_training_equals_the_device_table(dtype):
    m, twin, hf = _pair("maxpool", "hot", dtype=dtype, cls="sup", fused_pool=True)
    for s in range(5):                                  # the bf16 operand table must follow every step's working set
        ids, lab = _ids(s), _labels(s, False)
        assert torch.equal(m.train_step(ids, lab), twin.train_step(ids, lab)), s
        assert _same_params(m, twin), s


@pytest.mark.parametrize("kind,fused", [("mean", False), ("maxpool", True)])
def test_unsupervised_training_equals_the_device_table(kind, fused):
    m, twin, hf = _pair(kind, "hot", cls="unsup", fused_pool=fused)
    for s in range(5):
        b1, b2 = _ids(s), _ids(s + 50)
        assert torch.equal(m.train_step(b1, b2), twin.train_step(b1, b2)), s
        assert _same_params(m, twin), s
    assert float(m.mrr()) == float(twin.mrr())


def test_unsupervised_fused_pool_refuses_a_bf16_host_table():
    import graphsage_b200 as gs
    adj, feats = _data()
    hf = gs.HostFeatures(torch.from_numpy(feats).to(torch.bfloat16))
    with pytest.raises(NotImplementedError, match="bfloat16 host-memory"):
        _build("maxpool", hf, adj, cls="unsup", fused_pool=True)


# ------------------------------------------------------------------ capture
@pytest.mark.parametrize("kind", ["mean", "maxpool"])
def test_graphed_forward_replays_equal_eager_and_the_twin(kind):
    m, twin, hf = _pair(kind, "hot")
    eager, _, _ = _pair(kind, "hot")
    g = _first(m.graphed, B)
    for s in range(4):
        out = g(_ids(s).cuda()).clone()
        assert torch.equal(out, (_first if s == 0 else lambda f, x: f(x))(eager.forward, _ids(s))), s
        assert torch.equal(out, (_first if s == 0 else lambda f, x: f(x))(twin.forward, _ids(s))), s
    g.close()


@pytest.mark.parametrize("cls,kind", [("sup", "mean"), ("sup", "maxpool"), ("unsup", "mean")])
def test_graphed_train_step_replays_equal_eager_and_the_twin(cls, kind):
    import graphsage_b200 as gs
    m, twin, hf = _pair(kind, "hot", cls=cls)
    eager, _, _ = _pair(kind, "hot", cls=cls)
    gs.make_adam_capturable(twin.optimizer)
    gs.make_adam_capturable(eager.optimizer)
    step = m.graphed_train_step(B)
    for s in range(4):
        a = (_ids(s), _labels(s, False)) if cls == "sup" else (_ids(s), _ids(s + 50))
        loss = step(*[x.cuda() for x in a])
        assert torch.equal(loss, eager.train_step(*a)), s
        assert torch.equal(loss, twin.train_step(*a)), s
        assert _same_params(m, twin) and _same_params(m, eager), s


def test_a_step_does_not_synchronise():
    m, twin, hf = _pair("mean", "hot", cls="sup")
    ids, lab = _ids(0).cuda(), _labels(0, False).cuda()
    m.train_step(ids, lab)                              # lazy allocations and packs first
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        m.train_step(ids, lab)
        m.forward(ids)
    finally:
        torch.cuda.set_sync_debug_mode("default")


def test_pipelined_forward_is_refused():
    m, twin, hf = _pair("mean", "hot")
    with pytest.raises(NotImplementedError, match="PipelinedForward with a host-memory"):
        m.pipelined(B)


# ------------------------------------------------------------------ device memory
def test_device_memory_is_the_working_set_not_the_table():
    import graphsage_b200 as gs
    n, F, b = 1_000_000, 128, 256
    rs = np.random.RandomState(0)
    table = torch.from_numpy(rs.rand(n + 1, F).astype(np.float32))
    table[n] = 0
    adj = torch.from_numpy(rs.randint(0, n, size=(n + 1, 16)).astype(np.int32)).cuda()
    cache = np.arange(0, n, 10)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    hf = gs.HostFeatures(table, cache_ids=cache)
    sampler = gs.UniformNeighborSampler(adj, seed=1)
    infos = [gs.SAGEInfo("node", sampler, 10, 32), gs.SAGEInfo("node", sampler, 5, 32)]
    m = gs.SupervisedGraphsage(4, {"batch_size": b, "dropout": 0.}, hf, adj, None, infos, aggregator_type="mean")
    torch.cuda.synchronize()
    grown = torch.cuda.memory_allocated() - base
    S = b * (1 + 5 + 50)
    want = (len(cache) + 1 + S) * gs.ops.pad_cols(F) * 4 + 2 * (n + 1) * 4        # working set + cache map + claim array
    assert hf.capacity == S
    assert want <= grown <= want + (4 << 20), (grown, want)
    assert grown < table.numel() * 4 / 4
    m.train_step(torch.arange(b, dtype=torch.int32), torch.zeros((b, 4)))
    torch.cuda.synchronize()
    hf.close()


def test_toy_ppi_training_losses_equal_the_device_table():
    """The toy-ppi slice (tests/golden/toy_ppi.npz), supervised graphsage_mean with the sigmoid loss: every loss of a model
    on a HostFeatures table (its hottest third cached) is the device-table twin's, bit for bit."""
    import os
    import graphsage_b200 as gs
    from conftest import GOLDEN
    from graphsage_b200.host_features import hot_rows
    from graphsage_b200.minibatch import padded_from_csr_fast
    d = np.load(os.path.join(GOLDEN, "toy_ppi.npz"))
    n = d["feats"].shape[0]
    src, dst = np.concatenate([d["src"], d["dst"]]), np.concatenate([d["dst"], d["src"]])
    order = np.argsort(src, kind="stable")
    indptr = np.concatenate([[0], np.cumsum(np.bincount(src, minlength=n))]).astype(np.int64)
    adj, _ = padded_from_csr_fast(indptr, dst[order].astype(np.int32), 32, seed=1)
    feats = np.vstack([d["feats"].astype(np.float32), np.zeros((1, d["feats"].shape[1]), np.float32)])
    labels = torch.from_numpy(d["labels"].astype(np.float32))

    def build(features):
        gs.inits.manual_seed(3)
        adj_d = torch.from_numpy(adj).cuda()
        sampler = gs.UniformNeighborSampler(adj_d, seed=123)
        infos = [gs.SAGEInfo("node", sampler, 25, 64), gs.SAGEInfo("node", sampler, 10, 64)]
        return gs.SupervisedGraphsage(labels.shape[1], {"batch_size": 64, "dropout": 0.}, features, adj_d, None,
                                      infos, aggregator_type="mean", sigmoid_loss=True, learning_rate=0.01)
    hf = gs.HostFeatures(feats, cache_ids=hot_rows(adj, n // 3))
    m, twin = build(hf), build(torch.from_numpy(feats).cuda())
    rs = np.random.RandomState(0)
    for step in range(20):
        ids = rs.randint(0, n, size=64)
        batch, lab = torch.from_numpy(ids.astype(np.int32)), labels[torch.from_numpy(ids)]
        assert torch.equal(m.train_step(batch, lab), twin.train_step(batch, lab)), step
    assert _same_params(m, twin)
