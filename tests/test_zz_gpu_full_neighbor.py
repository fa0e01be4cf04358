"""GPU: full-neighbourhood inference.  gs_csr_aggregate bit for bit against oracle/full_neighbor.py and against the
fixed-fanout kernels (gs_gather_mean, gs_segment_max) on a CSR built from a fixed-fanout sample;
SampleAndAggregate.full_neighbor_embeddings against the oracle's layer loop (1e-4 relative, test_gpu_parity's TOL),
its determinism, subsets, agreement with forward() where sampling draws whole rows, a toy-ppi run through
full_neighbor_predict, and the refusals."""
import numpy as np
import pytest
import torch

from conftest import load_golden, rel_err
from oracle import full_neighbor as fn
from oracle import numerics as nu

pytestmark = pytest.mark.gpu
TOL = 1e-4


@pytest.fixture(scope="module")
def gs():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    import graphsage_b200
    graphsage_b200._lib.lib()
    return graphsage_b200


def dev(x):
    return torch.as_tensor(np.ascontiguousarray(x)).cuda()


def edge_csr(rs, n_nodes, n_src):
    """Degrees 0, 1, 31, 32, 33, 257 (a hub-role row) and random ones; duplicates, self loops, out-of-range entries."""
    deg = rs.randint(0, 40, size=n_nodes)
    deg[:7] = [0, 1, 31, 32, 33, 257, 600]
    indptr = np.concatenate([[0], np.cumsum(deg)]).astype(np.int64)
    indices = rs.randint(0, n_src, size=int(indptr[-1])).astype(np.int32)
    indices[indptr[1]] = 1                                              # node 1's only entry: a self loop
    indices[indptr[2]:indptr[2] + 5] = 7                                # duplicates
    bad = rs.rand(len(indices)) < 0.02
    indices[bad] = rs.choice([-1, -7, n_src, n_src + 3], size=int(bad.sum()))
    return indptr, indices


def table_of(rs, n_src, F, dtype):
    """(device view [n_src, F] with poisoned pad columns - a 16-byte pitch, or an odd one for "fp32_odd" - and the
    oracle's fp32 table, bf16-rounded for "bf16")."""
    x = rs.randn(n_src, F).astype(np.float32)
    if dtype == "bf16":
        t = torch.full((n_src, (F + 7) // 8 * 8), 7.0, device="cuda")
        t[:, :F] = dev(x)
        tb = t.to(torch.bfloat16)
        return tb[:, :F], tb[:, :F].float().cpu().numpy()
    pitch = (F + 7) // 8 * 8 if dtype == "fp32" else (F + 1 if F % 2 == 0 else F + 2)
    t = torch.full((n_src, pitch), 7.0, device="cuda")
    t[:, :F] = dev(x)
    return t[:, :F], x


@pytest.mark.parametrize("dtype", ["fp32", "fp32_odd", "bf16"])
@pytest.mark.parametrize("F", [1, 5, 602, 1024])
@pytest.mark.parametrize("op", fn.OPS)
def test_csr_aggregate_bit_exact(gs, op, F, dtype):
    rs = np.random.RandomState(F)
    n_nodes, n_src = 120, 140
    indptr, indices = edge_csr(rs, n_nodes, n_src)
    src, ref_table = table_of(rs, n_src, F, dtype)
    for rows in (None, np.array([3, 0, 5, -2, n_nodes, n_nodes + 40, 6, 5, 119], dtype=np.int32)):
        got = gs.ops.csr_aggregate(src, dev(indptr), dev(indices), op, rows=None if rows is None else dev(rows))
        want = fn.csr_aggregate(ref_table, indptr, indices, op, rows)
        assert nu.bits_equal(got.cpu().numpy(), want), (op, F, dtype, rows is None)
        buf = got.as_strided((got.shape[0], gs.ops.pad_cols(F)), (got.stride(0), 1))
        assert (buf[:, F:] == 0).all()                                  # pad columns zeroed


@pytest.mark.parametrize("op", fn.OPS)
def test_a_row_of_1e5_entries(gs, op):
    rs = np.random.RandomState(9)
    n_src, F = 3000, 602
    x = rs.randn(n_src, F).astype(np.float32)
    indptr = np.array([0, 3, 100003, 100010], dtype=np.int64)
    indices = rs.randint(0, n_src, size=100010).astype(np.int32)
    got = gs.ops.csr_aggregate(dev(x), dev(indptr), dev(indices), op).cpu().numpy()
    want = fn.csr_aggregate(x, indptr, indices, op)
    assert nu.bits_equal(got, want)
    again = gs.ops.csr_aggregate(dev(x), dev(indptr), dev(indices), op).cpu().numpy()
    assert nu.bits_equal(got, again)


@pytest.mark.parametrize("k", [1, 25, 300])
@pytest.mark.parametrize("dtype", ["fp32", "bf16"])
def test_fixed_fanout_csr_equals_the_fanout_kernels(gs, k, dtype):
    rs = np.random.RandomState(k)
    n, n_src, F = 200, 500, 602
    src, _ = table_of(rs, n_src, F, dtype)
    ids = dev(rs.randint(-2, n_src + 2, size=n * k).astype(np.int32))
    selfs = dev(np.arange(n, dtype=np.int32))
    indptr = torch.arange(n + 1, dtype=torch.int64, device="cuda") * k
    for include_self in (False, True):
        _, mean = gs.ops.gather_mean(src, [gs.ops.Seg(n, k, self_ids=selfs, neigh_ids=ids)], include_self=include_self,
                                     want_self=False)
        got = gs.ops.csr_aggregate(src, indptr, ids, "mean_self" if include_self else "mean", rows=selfs)
        assert nu.bits_equal(got.cpu().numpy(), mean[:, :F].cpu().numpy()), (k, dtype, include_self)
    z = torch.relu(torch.randn((n_src, 512), device="cuda"))            # pooled MLP outputs: ReLU zeros included
    zs = torch.zeros((n_src, 512), device="cuda")
    zs.copy_(z)
    rows = gs.ops.gather_rows(zs, ids)
    want = gs.ops.segment_max(rows, n, k)
    got = gs.ops.csr_aggregate(zs, indptr, ids, "max", rows=selfs)
    assert nu.bits_equal(got.cpu().numpy(), want.cpu().numpy())


# ---------------------------------------------------------------- the model
def model_of(gs, kind, concat=True, math="fp32", table="fp32", identity_dim=0, layers=2, n=300, F=20, seed=0,
             adj=None, fanout=5):
    rs = np.random.RandomState(seed)
    feats = np.vstack([rs.randn(n, F).astype(np.float32), np.zeros((1, F), np.float32)])
    gs.set_default_math(math)
    gs.inits.manual_seed(seed + 1)
    if adj is None:
        adj = rs.randint(0, n, size=(n + 1, 8)).astype(np.int32)
        adj[n] = n
    adj = dev(adj)
    sampler = gs.UniformNeighborSampler(adj, seed=3)
    dims = [16, 12, 8][:layers]
    infos = [gs.SAGEInfo("node", sampler, fanout, d) for d in dims]
    f = dev(feats)
    if table == "bf16":
        f = f.to(torch.bfloat16)
    m = gs.SampleAndAggregate({"batch_size": 8, "dropout": 0.}, f, adj, None, infos, concat=concat, aggregator_type=kind,
                              identity_dim=identity_dim)
    gs.set_default_math("fp32")
    return m


def oracle_aggs(m):
    out = []
    for a in m.aggregators:
        d = {k: v.detach().cpu().numpy() for k, v in a.vars.items()}
        if hasattr(a, "mlp_layers"):
            d["mlp_weights"] = a.mlp_layers[0].vars["weights"].detach().cpu().numpy()
            d["mlp_bias"] = a.mlp_layers[0].vars["bias"].detach().cpu().numpy()
        d["type"] = {"MeanAggregator": "mean", "GCNAggregator": "gcn", "MaxPoolingAggregator": "maxpool",
                     "MeanPoolingAggregator": "meanpool"}[type(a).__name__]
        out.append(d)
    return out


def graph(seed, n=300):
    rs = np.random.RandomState(seed)
    return edge_csr(rs, n, n)


MODEL_CASES = ([(k, c, "fp32", "fp32", 0, 2) for k in ("mean", "maxpool", "meanpool") for c in (False, True)]
               + [("gcn", False, "fp32", "fp32", 0, 2),
                  ("mean", True, "tf32x3", "fp32", 0, 2), ("maxpool", True, "tf32x3", "fp32", 0, 2),
                  ("gcn", False, "tf32x3", "fp32", 0, 2),
                  ("mean", True, "fp32", "bf16", 0, 2), ("maxpool", False, "fp32", "bf16", 0, 2),
                  ("gcn", False, "fp32", "bf16", 0, 2), ("meanpool", True, "tf32x3", "bf16", 0, 2),
                  ("mean", True, "fp32", "fp32", 16, 2), ("maxpool", True, "fp32", "fp32", 16, 2),
                  ("gcn", False, "tf32x3", "fp32", 16, 2),
                  ("mean", True, "fp32", "fp32", 0, 3), ("maxpool", True, "tf32x3", "fp32", 0, 3),
                  ("gcn", False, "fp32", "fp32", 0, 3)])


@pytest.mark.parametrize("kind,concat,math,table,identity_dim,layers", MODEL_CASES)
def test_model_equals_the_oracle(gs, kind, concat, math, table, identity_dim, layers):
    m = model_of(gs, kind, concat, math, table, identity_dim, layers)
    indptr, indices = graph(1)
    got = m.full_neighbor_embeddings(dev(indptr), dev(indices))
    feats = m.features.float().cpu().numpy()                            # bf16-rounded / embeddings first, as the model reads it
    want = fn.full_neighbor_embeddings(feats, indptr, indices, oracle_aggs(m), concat)
    assert got.shape == want.shape
    assert rel_err(got.cpu().numpy(), want) < TOL
    ids = np.array([0, 5, 299, 17, 17, 300], dtype=np.int32)            # 300: the dummy node
    sub = m.full_neighbor_embeddings(indptr, indices, node_ids=ids)
    assert rel_err(sub.cpu().numpy(), fn.full_neighbor_embeddings(feats, indptr, indices, oracle_aggs(m), concat,
                                                                  node_ids=ids)) < TOL


@pytest.mark.parametrize("kind", ["mean", "gcn", "maxpool"])
def test_subsets_and_repeated_calls(gs, kind):
    m = model_of(gs, kind, concat=kind != "gcn", math="tf32x3")
    indptr, indices = (dev(a) for a in graph(2))
    full = m.full_neighbor_embeddings(indptr, indices)
    assert torch.equal(full, m.full_neighbor_embeddings(indptr, indices))
    ids = torch.tensor([7, 0, 299, 7, 150], dtype=torch.int32)
    sub = m.full_neighbor_embeddings(indptr, indices, node_ids=ids)
    assert torch.allclose(sub, full[ids.long().cuda()], rtol=1e-6, atol=1e-7)
    raw = m.full_neighbor_embeddings(indptr, indices, normalize=False)
    assert torch.allclose(torch.nn.functional.normalize(raw, dim=1), full, rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize("kind", ["mean", "gcn", "maxpool", "meanpool"])
def test_regular_graph_with_whole_row_samples_matches_forward(gs, kind):
    n, d = 200, 6
    rs = np.random.RandomState(4)
    indices = np.concatenate([rs.choice(n, d, replace=False) for _ in range(n)]).astype(np.int32)
    indptr = np.arange(n + 1, dtype=np.int64) * d
    adj = np.full((n + 1, d), n, dtype=np.int32)
    for v in range(n):
        adj[v] = rs.permutation(indices[v * d:(v + 1) * d])
    m = model_of(gs, kind, concat=kind != "gcn", n=n, adj=adj, fanout=d)
    ids = torch.arange(n, dtype=torch.int32)
    fwd = m.forward(ids).cpu().numpy()
    got = m.full_neighbor_embeddings(indptr, indices).cpu().numpy()
    assert rel_err(got, fwd) < TOL


def test_toy_ppi_full_neighbor_predict(gs):
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
    gs.inits.manual_seed(3)
    sampler = gs.UniformNeighborSampler(dev(it.adj), seed=1)
    infos = [gs.SAGEInfo("node", sampler, 10, 64), gs.SAGEInfo("node", sampler, 5, 64)]
    m = gs.SupervisedGraphsage(labels.shape[1], {"batch_size": 64, "dropout": 0.}, feats, dev(it.adj), None, infos,
                               aggregator_type="mean", sigmoid_loss=True, learning_rate=0.01)
    train = np.array([id2idx[u] for u in G.nodes() if not G.node[u]["val"] and not G.node[u]["test"]])
    rs = np.random.RandomState(0)
    for _ in range(20):
        ids = rs.choice(train, 64).astype(np.int32)
        m.train_step(torch.from_numpy(ids), torch.from_numpy(labels[ids]))
    val = np.array([id2idx[u] for u in G.nodes() if G.node[u]["val"]], dtype=np.int32)
    indptr, indices = it.neighbor_csr(test=True)
    preds = m.full_neighbor_predict(indptr, indices, val)
    assert preds.shape == (len(val), labels.shape[1])
    again = m.full_neighbor_predict(indptr, indices, val)
    assert torch.equal(preds, again)
    f1_micro, f1_macro = calc_f1(labels[val], preds.cpu().numpy(), True)
    print("toy-ppi full-neighbourhood val F1 micro %.4f macro %.4f" % (f1_micro, f1_macro))
    assert 0.0 < f1_micro <= 1.0 and np.isfinite(f1_macro)


def test_refusals(gs):
    m = model_of(gs, "mean")
    indptr, indices = graph(5)
    with pytest.raises(ValueError, match="indptr is on cpu"):
        m.full_neighbor_embeddings(torch.from_numpy(indptr), dev(indices))
    with pytest.raises(ValueError, match="indices is on cpu"):
        m.full_neighbor_embeddings(dev(indptr), torch.from_numpy(indices))
    with pytest.raises(TypeError, match="indptr"):
        m.full_neighbor_embeddings(dev(indptr.astype(np.int32)), dev(indices))
    with pytest.raises(TypeError, match="indices"):
        m.full_neighbor_embeddings(dev(indptr), dev(indices.astype(np.int64)))
    with pytest.raises(ValueError, match="N \\+ 1"):
        m.full_neighbor_embeddings(dev(indptr[:-1]), dev(indices))
    seq = model_of(gs, "seq")
    with pytest.raises(NotImplementedError, match="seq"):
        seq.full_neighbor_embeddings(indptr, indices)
    with pytest.raises(ValueError, match="op"):
        gs.ops.csr_aggregate(m.features, dev(indptr), dev(indices), "sum")
