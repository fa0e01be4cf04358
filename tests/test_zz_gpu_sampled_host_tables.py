"""GPU: sampled blocks over host-memory and int8 feature tables.  The layer-0 loader (gs_host_gather_rows_f32) byte for
byte against tests/host_gather_ref.py; sampled embeddings, losses, gradients and Adam steps torch.equal to the twin on
the device table for every table kind; one host synchronisation per loss and backward; peak device memory on a
1,000,000-row host table; a toy-ppi epoch on a host int8 table."""
import gc
import warnings

import numpy as np
import pytest
import torch

from conftest import load_golden
from host_gather_ref import gather_rows_f32 as ref_gather
from test_zz_gpu_full_neighbor import dev, edge_csr

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def gs():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    import graphsage_b200
    graphsage_b200._lib.lib()
    return graphsage_b200


def _feats(n, F, seed=0):
    rs = np.random.RandomState(seed)
    x = (rs.randn(n + 1, F) * rs.uniform(0.05, 4, size=(n + 1, 1))).astype(np.float32)
    x[n] = 0
    return x


def _host_table(gs, dtype, x, cache_ids):
    if dtype == "fp32":
        return gs.HostFeatures(x, cache_ids=cache_ids)
    if dtype == "bf16":
        return gs.HostFeatures(torch.from_numpy(x).to(torch.bfloat16), cache_ids=cache_ids)
    return gs.HostFeatures(gs.Int8Features(x), cache_ids=cache_ids)


def _stored(t, dtype):
    """A CPU tensor of stored rows as the restatement takes them."""
    t = t.cpu()
    return t.view(torch.int16).numpy().view(np.uint16) if dtype == "bf16" else t.numpy()


KIND = {"fp32": "f32", "bf16": "bf16", "int8": "i8row"}


# ---------------------------------------------------------------- the loader, byte for byte
@pytest.mark.parametrize("cache", ["none", "some", "all"])
@pytest.mark.parametrize("F", [1, 3, 50, 602, 1536, 4100])   # int8 rows past 4,092 take the flat walk
@pytest.mark.parametrize("dtype", ["fp32", "bf16", "int8"])
def test_loader_bytes_equal_the_restatement(gs, dtype, F, cache):
    n = 300
    x = _feats(n, F, seed=F)
    cache_ids = {"none": None, "some": np.arange(0, n, 7), "all": np.arange(n)}[cache]
    h = _host_table(gs, dtype, x, cache_ids)
    C = h.n_cached
    if C:      # the cached rows are given other bytes than the host's: the rule, not the values, picks the source
        h.ws[:C] = h.host[torch.from_numpy(np.asarray(cache_ids)[::-1].copy())].to(h.ws.device)
    rs = np.random.RandomState(F + C)
    ids = np.concatenate([rs.randint(0, n, size=500), [5, 5, 5, n, -1, -7, n + 1, 2**31 - 1, 0, n - 1]])
    rs.shuffle(ids)
    ids = dev(ids.astype(np.int32))
    pad = gs.ops.pad_cols(F)
    buf = torch.full((ids.numel(), pad), float("nan"), device="cuda")
    got = gs.ops.host_gather_rows_f32(h._alias, h.ws, h.cache_slot, n, F, ids, out=buf[:, :F])
    assert got.data_ptr() == buf.data_ptr()
    want = ref_gather(_stored(h.host, dtype), _stored(h.ws[:C], dtype), h.cache_slot.cpu().numpy(), ids.cpu().numpy(), F,
                      KIND[dtype])
    assert np.array_equal(buf.cpu().numpy().view(np.uint32), want.view(np.uint32))
    # the method: the [:, :F] view of a pad_cols(F) buffer, as gather_rows_f32 lays it out
    m = h.gather_rows_f32(ids)
    assert m.shape == (ids.numel(), F) and m.stride(0) == pad and torch.equal(m, buf[:, :F])
    assert h.gather_rows_f32(dev(np.zeros(0, np.int32))).shape == (0, F)
    h.close()


@pytest.mark.parametrize("dtype", ["fp32", "bf16", "int8"])
def test_device_twin_rows_and_a_grid_that_loops(gs, dtype):
    """On the uncorrupted table the rows are gather_rows_f32's on the device table; a list longer than one pass of the
    capped grid (3 CTAs x 256 threads x 8 loads per SM) is read whole."""
    n, F = 500, 3
    x = _feats(n, F, seed=1)
    h = _host_table(gs, dtype, x, np.arange(0, n, 3))
    device = {"fp32": lambda: dev(x), "bf16": lambda: dev(x).to(torch.bfloat16),
              "int8": lambda: gs.Int8Features(x, device="cuda")}[dtype]()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    total = sms * 3 * 256 * 8 * 2 + 777            # F = 3: one output unit per row for bf16 / int8, two for fp32
    ids = dev(np.random.RandomState(2).randint(-3, n + 3, size=total).astype(np.int32))
    got = h.gather_rows_f32(ids)
    assert torch.equal(got, gs.ops.gather_rows_f32(device, ids))
    want = ref_gather(_stored(h.host, dtype), _stored(h.ws[:h.n_cached], dtype), h.cache_slot.cpu().numpy(),
                      ids.cpu().numpy(), F, KIND[dtype])
    assert np.array_equal(got.cpu().numpy(), want[:, :F])
    h.close()


def test_loader_argument_checks(gs):
    h = _host_table(gs, "fp32", _feats(10, 4), None)
    ids = dev(np.arange(5, dtype=np.int32))
    with pytest.raises(RuntimeError, match="out_pitch"):
        gs.ops.host_gather_rows_f32(h._alias, h.ws, h.cache_slot, 10, 4, ids,
                                    out=torch.empty((5, 6), device="cuda")[:, :4])
    with pytest.raises(TypeError, match="ids must be int32"):
        gs.ops.host_gather_rows_f32(h._alias, h.ws, h.cache_slot, 10, 4, ids.long())
    h.close()
    h = _host_table(gs, "int8", _feats(10, 4), None)             # int8 rows cover gs_i8row_pitch(4) = 16 columns
    with pytest.raises(RuntimeError, match="out_pitch <= gs_i8row_pitch"):
        gs.ops.host_gather_rows_f32(h._alias, h.ws, h.cache_slot, 10, 4, ids,
                                    out=torch.empty((5, 32), device="cuda")[:, :4])
    h.close()


# ---------------------------------------------------------------- models: torch.equal to the device twin
TWINS = ["host-fp32", "host-fp32-cached", "host-bf16", "host-int8", "host-int8-cached", "int8-fp32", "host-int8-fp32"]


def _twin_tables(gs, twin, x, cache_ids):
    """(the table under test, its twin's table on the device)."""
    cache = cache_ids if twin.endswith("cached") else None
    if twin.startswith("host-fp32"):
        return _host_table(gs, "fp32", x, cache), dev(x)
    if twin == "host-bf16":
        return _host_table(gs, "bf16", x, cache_ids), dev(x).to(torch.bfloat16)
    if twin.startswith("host-int8"):
        d = gs.Int8Features(x, device="cuda")
        return _host_table(gs, "int8", x, cache), d.dequantize() if twin.endswith("fp32") else d
    d = gs.Int8Features(x, device="cuda")                # "int8-fp32": the device int8 table against its dequantize()
    return d, d.dequantize()


def _model(gs, features, adj, agg, concat, math, layers, unsup=False, fanout=5):
    gs.set_default_math(math)
    gs.inits.manual_seed(11)
    sampler = gs.UniformNeighborSampler(adj, seed=3)
    infos = [gs.SAGEInfo("node", sampler, fanout, d) for d in [16, 12, 8][:layers]]
    try:
        if unsup:
            return gs.UnsupervisedGraphsage({"batch_size": 8, "dropout": 0.}, features, adj,
                                            np.random.RandomState(0).randint(1, 9, size=adj.shape[0] - 1), infos,
                                            concat=concat, aggregator_type=agg, neg_sample_size=6, weight_decay=0.01,
                                            learning_rate=0.01)
        return gs.SupervisedGraphsage(4, {"batch_size": 8, "dropout": 0.}, features, adj, None, infos, concat=concat,
                                      aggregator_type=agg, weight_decay=0.01)
    finally:
        gs.set_default_math("fp32")


def _graph(n=300):
    rs = np.random.RandomState(1)
    indptr, indices = edge_csr(rs, n, n)
    adj = rs.randint(0, n, size=(n + 1, 8)).astype(np.int32)
    adj[n] = n
    return dev(indptr), dev(indices), dev(adj)


def _sup_run(m, indptr, indices, ids, labels, dropout=None, train=True):
    emb = m.sampled_minibatch_embeddings(indptr, indices, ids)
    if not train:
        return [emb]
    m.optimizer.zero_grad(set_to_none=True)
    out = m.sampled_minibatch_outputs(indptr, indices, ids, dropout=dropout)
    loss = m.sampled_minibatch_loss(indptr, indices, ids, labels, dropout=dropout)
    loss.backward()
    grads = [p.grad.clone() for p in m.parameters()]
    steps = [m.sampled_minibatch_train_step(indptr, indices, ids, labels, dropout=dropout) for _ in range(5)]
    return [emb, out.detach(), loss.detach()] + grads + steps + [p.detach().clone() for p in m.parameters()]


def _unsup_run(m, indptr, indices, b1, b2):
    emb = m.sampled_minibatch_embeddings(indptr, indices, b1)
    m.optimizer.zero_grad(set_to_none=True)
    loss = m.sampled_minibatch_loss(indptr, indices, b1, b2)
    loss.backward()
    grads = [p.grad.clone() for p in m.parameters()]
    steps = [m.sampled_minibatch_train_step(indptr, indices, b1, b2) for _ in range(5)]
    return [emb, loss.detach()] + grads + steps + [p.detach().clone() for p in m.parameters()]


def _assert_same(a, b):
    assert len(a) == len(b)
    for i, (x, y) in enumerate(zip(a, b)):
        assert x.shape == y.shape and torch.equal(x, y), i


IDS = np.array([0, 5, 299, 17, 17, 4, 150, 6, 1, 2, 3, -1, 300, 5], dtype=np.int32)
LABELS = np.eye(4, dtype=np.float32)[np.arange(len(IDS)) % 4]


@pytest.mark.parametrize("twin", TWINS)
@pytest.mark.parametrize("agg,concat,math,layers", [
    ("mean", True, "fp32", 2), ("mean", False, "tf32x3", 3), ("gcn", False, "fp32", 2), ("gcn", False, "tf32x3", 1),
    ("maxpool", True, "tf32x3", 2), ("maxpool", False, "fp32", 1), ("meanpool", True, "fp32", 3),
    ("meanpool", False, "tf32x3", 2)])
def test_supervised_equals_the_device_twin(gs, twin, agg, concat, math, layers):
    indptr, indices, adj = _graph()
    x = _feats(300, 50, seed=4)
    t, d = _twin_tables(gs, twin, x, np.arange(0, 300, 3))
    a = _sup_run(_model(gs, t, adj, agg, concat, math, layers), indptr, indices, IDS, LABELS)
    b = _sup_run(_model(gs, d, adj, agg, concat, math, layers), indptr, indices, IDS, LABELS)
    _assert_same(a, b)


@pytest.mark.parametrize("twin", ["host-fp32", "host-bf16", "host-int8-cached", "int8-fp32"])
def test_twomaxpool_embeddings_equal_the_device_twin(gs, twin):
    indptr, indices, adj = _graph()
    t, d = _twin_tables(gs, twin, _feats(300, 50, seed=5), np.arange(0, 300, 3))
    for concat, layers in ((True, 2), (False, 1)):
        a = _sup_run(_model(gs, t, adj, "twomaxpool", concat, "tf32x3", layers), indptr, indices, IDS, None, train=False)
        b = _sup_run(_model(gs, d, adj, "twomaxpool", concat, "tf32x3", layers), indptr, indices, IDS, None, train=False)
        _assert_same(a, b)


@pytest.mark.parametrize("twin", ["host-fp32-cached", "host-bf16", "host-int8", "int8-fp32"])
@pytest.mark.parametrize("agg,math", [("mean", "fp32"), ("gcn", "tf32x3"), ("maxpool", "fp32"), ("meanpool", "tf32x3")])
def test_unsupervised_equals_the_device_twin(gs, twin, agg, math):
    indptr, indices, adj = _graph()
    t, d = _twin_tables(gs, twin, _feats(300, 20, seed=6), np.arange(0, 300, 4))
    b1, b2 = dev(np.array([1, 2, 3, 9, 40], np.int32)), dev(np.array([4, 4, 38, 0, 299], np.int32))
    a = _unsup_run(_model(gs, t, adj, agg, agg != "gcn", math, 2, unsup=True), indptr, indices, b1, b2)
    b = _unsup_run(_model(gs, d, adj, agg, agg != "gcn", math, 2, unsup=True), indptr, indices, b1, b2)
    _assert_same(a, b)


@pytest.mark.parametrize("twin", ["host-fp32-cached", "host-bf16"])
@pytest.mark.parametrize("agg,math", [("mean", "fp32"), ("gcn", "tf32x3"), ("maxpool", "tf32x3"), ("meanpool", "fp32")])
def test_host_dropout_equals_the_device_twin(gs, twin, agg, math):
    indptr, indices, adj = _graph()
    t, d = _twin_tables(gs, twin, _feats(300, 50, seed=7), np.arange(0, 300, 2))
    ma, mb = (_model(gs, f, adj, agg, agg != "gcn", math, 2) for f in (t, d))
    a = _sup_run(ma, indptr, indices, IDS, LABELS, dropout=0.5)
    b = _sup_run(mb, indptr, indices, IDS, LABELS, dropout=0.5)
    _assert_same(a, b)
    assert ma.dropout_counter == mb.dropout_counter > 0
    with pytest.raises(NotImplementedError, match="torch.int8"):
        _model(gs, gs.Int8Features(_feats(300, 50), device="cuda"), adj, agg, True, math, 2).sampled_minibatch_loss(
            indptr, indices, IDS, LABELS, dropout=0.5)


def test_whole_graph_entry_points_still_refuse(gs):
    indptr, indices, adj = _graph()
    for t in _twin_tables(gs, "host-fp32", _feats(300, 8), None)[:1] + (gs.Int8Features(_feats(300, 8), device="cuda"),):
        m = _model(gs, t, adj, "mean", True, "fp32", 2)
        with pytest.raises(NotImplementedError, match="full-neighbourhood"):
            m.full_neighbor_minibatch_embeddings(indptr, indices, IDS)
        with pytest.raises(NotImplementedError, match="full-neighbourhood"):
            m.full_neighbor_loss(indptr, indices, IDS, LABELS)


# ---------------------------------------------------------------- host reads and memory
@pytest.mark.parametrize("twin", ["host-fp32-cached", "host-int8", "int8"])
def test_one_host_synchronisation_per_loss_and_backward(gs, twin):
    indptr, indices, adj = _graph()
    t, _ = _twin_tables(gs, twin, _feats(300, 50), np.arange(0, 300, 5))
    m = _model(gs, t, adj, "maxpool", True, "tf32x3", 2)
    ids, labels = dev(IDS), dev(LABELS)
    m.sampled_minibatch_loss(indptr, indices, ids, labels).backward()          # lazy set-up
    gc.collect()           # an earlier test's HostFeatures synchronises when it is closed: not inside the counted call
    torch.cuda.set_sync_debug_mode("warn")        # the first switch of the mode in a process reports a sync of its own
    torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            m.sampled_minibatch_loss(indptr, indices, ids, labels).backward()
        finally:
            torch.cuda.set_sync_debug_mode("default")
    syncs = [x for x in w if "synchroniz" in str(x.message)]
    reads = len(syncs)
    print("host synchronisations per sampled loss + backward on a %s table: %d (%s)"
          % (twin, reads, ", ".join("%s:%d" % (x.filename.split("/")[-1], x.lineno) for x in syncs)))
    assert reads == 1


def test_peak_memory_on_a_million_row_host_table(gs):
    """One sampled step on a 1,000,000 x 128 fp32 host table (nothing cached): the device holds the CSR, the cache map
    and block-sized buffers.  Bound: the block build's workspace + 3 fp32 rows of pad_cols(F) per node of V_0 (X0 is
    the one layer-0 buffer that size) + 32 MB."""
    from graphsage_b200 import ops
    n, F, batch = 1000000, 128, 512
    rs = np.random.RandomState(9)
    x = np.zeros((n + 1, F), np.float32)
    x[:n] = rs.randn(n, F)
    deg = rs.randint(0, 20, size=n)
    indptr = dev(np.concatenate([[0], np.cumsum(deg)]).astype(np.int64))
    indices = dev(rs.randint(0, n, size=int(deg.sum())).astype(np.int32))
    adj = dev(np.full((n + 1, 1), n, np.int32))
    h = gs.HostFeatures(x, cache_ids=None)
    del x
    gs.inits.manual_seed(1)
    sampler = gs.UniformNeighborSampler(adj, seed=3)
    infos = [gs.SAGEInfo("node", sampler, k, 128) for k in (25, 10)]
    m = gs.SupervisedGraphsage(8, {"dropout": 0.}, h, adj, None, infos, aggregator_type="mean")
    ids = dev(rs.randint(0, n, size=batch).astype(np.int32))
    labels = dev(np.eye(8, dtype=np.float32)[np.arange(batch) % 8])
    m.sampled_minibatch_train_step(indptr, indices, ids, labels)                # lazy set-up, Adam state
    blocks = ops.csr_blocks(indptr, indices, ids, 2, fanouts=[25, 10], seed=sampler.seed, call=sampler.counter)
    v0 = blocks[0].src_ids.numel()
    del blocks
    ws = gs._lib.lib().gs_csr_blocks_workspace_bytes(n, int(indices.numel()), batch, 2)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    m.sampled_minibatch_train_step(indptr, indices, ids, labels)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    bound = ws + 3 * v0 * ops.pad_cols(F) * 4 + (32 << 20)
    table = (n + 1) * F * 4
    print("1M x 128 host table: |V_0| = %d, step peak %.1f MB over the resident %.1f MB, bound %.1f MB, table %.1f MB"
          % (v0, peak / 2**20, base / 2**20, bound / 2**20, table / 2**20))
    assert peak <= bound and peak < table / 4
    h.close()


def test_toy_ppi_epoch_on_a_host_int8_table(gs):
    from test_walks_cpu import toy_graph
    from graphsage_b200.host_features import hot_rows
    from graphsage_b200.minibatch import NodeMinibatchIterator
    g = load_golden("toy_ppi")
    G = toy_graph()
    id2idx = {u: i for i, u in enumerate(G.nodes())}
    labels = (np.asarray(g["labels"]) > 0).astype(np.float32)
    it = NodeMinibatchIterator(G, id2idx, None, {u: labels[i] for i, u in enumerate(G.nodes())}, labels.shape[1],
                               batch_size=64, max_degree=25, rng=np.random.RandomState(0))
    n = len(id2idx)
    feats = np.zeros((n + 1, 50), np.float32)
    feats[:n] = np.asarray(g["feats"], np.float32)
    train = np.array([id2idx[u] for u in G.nodes() if not G.node[u]["val"] and not G.node[u]["test"]], dtype=np.int32)
    np_ptr, np_idx = it.neighbor_csr(test=False)
    tr_ptr, tr_idx = dev(np_ptr), dev(np_idx)
    d_lab = dev(labels)
    order = np.random.RandomState(0).permutation(train)
    tables = {"host": gs.HostFeatures(gs.Int8Features(feats), cache_ids=hot_rows((np_ptr, np_idx), n // 3)),
              "device": gs.Int8Features(feats, device="cuda")}
    assert 0 < tables["host"].n_cached <= n // 3
    losses = {}
    for name, t in tables.items():
        gs.inits.manual_seed(3)
        sampler = gs.UniformNeighborSampler(dev(it.adj), seed=1)
        infos = [gs.SAGEInfo("node", sampler, 10, 64), gs.SAGEInfo("node", sampler, 5, 64)]
        m = gs.SupervisedGraphsage(labels.shape[1], {"dropout": 0.}, t, dev(it.adj), None, infos,
                                   aggregator_type="mean", sigmoid_loss=True, learning_rate=0.03)
        losses[name] = torch.stack([m.sampled_minibatch_train_step(tr_ptr, tr_idx, dev(order[i:i + 512]),
                                                                   d_lab[dev(order[i:i + 512]).long()])
                                    for i in range(0, len(order), 512)])
    s = losses["host"].cpu().numpy()
    print("toy-ppi one epoch of 512-node steps on a host int8 table (a third cached): loss %.4f -> %.4f over %d steps"
          % (s[0], s[-1], len(s)))
    assert torch.equal(losses["host"], losses["device"])
    assert np.all(np.isfinite(s)) and s[-1] < s[0]
