"""Full-neighbourhood inference on the CPU: oracle/full_neighbor.py against the reference-written fixture
(tests/golden/full_neighbor.npz) and against a float64 dense-adjacency formula, its empty-row / dummy / clamp rules,
_TableOwner.neighbor_csr against the rows behind construct_adj / construct_test_adj, and the refusals."""
import numpy as np
import pytest
import torch

from conftest import load_golden

from graphsage_b200 import ops
from graphsage_b200.aggregators import MeanAggregator, SeqAggregator
from graphsage_b200.graph import to_csr
from graphsage_b200.minibatch import NodeMinibatchIterator
from graphsage_b200.models import SampleAndAggregate
from oracle import full_neighbor as fn
from oracle import numerics as nu

FX = load_golden("full_neighbor")


def fixture_aggs(name):
    aggs = []
    for li in range(2):
        prefix = "%s_L%d_" % (name, li)
        d = {k[len(prefix):]: FX[k] for k in FX.files if k.startswith(prefix)}
        d["type"] = name.split("_")[0]
        aggs.append(d)
    return aggs


@pytest.mark.parametrize("name", [str(c) for c in FX["cases"]])
def test_oracle_equals_the_reference_fixture(name):
    got = fn.full_neighbor_embeddings(FX["feats"], FX["indptr"], FX["indices"], fixture_aggs(name),
                                      bool(FX[name + "_concat"]))
    ref = FX[name + "_out"]
    assert got.shape == ref.shape
    assert np.abs(got - ref).max() <= 1e-5 * max(1.0, np.abs(ref).max()), name


def random_csr(rs, n_nodes, n_src, max_deg, bad=True):
    deg = rs.randint(0, max_deg + 1, size=n_nodes)
    deg[: min(3, n_nodes)] = [0, 1, max_deg][: min(3, n_nodes)]
    indptr = np.concatenate([[0], np.cumsum(deg)]).astype(np.int64)
    lo, hi = (-3, n_src + 3) if bad else (0, n_src)
    indices = rs.randint(lo, hi, size=int(indptr[-1])).astype(np.int32)
    return indptr, indices


@pytest.mark.parametrize("op", fn.OPS)
@pytest.mark.parametrize("rows", [None, "subset"])
def test_csr_aggregate_equals_the_dense_formula(op, rows):
    rs = np.random.RandomState(3)
    n_nodes, n_src, F = 60, 75, 9
    indptr, indices = random_csr(rs, n_nodes, n_src, 40)
    table = rs.randn(n_src, F).astype(np.float32)
    r = None if rows is None else np.array([5, 0, -1, n_nodes, n_nodes + 7, 2, 2, 59], dtype=np.int32)
    got = fn.csr_aggregate(table, indptr, indices, op, r)
    ref = fn.dense_reference(table, indptr, indices, op, r)
    assert got.shape == (n_nodes + 1 if r is None else len(r), F)
    assert np.allclose(got, ref, rtol=1e-5, atol=1e-6)


def test_empty_rows_dummy_node_and_clamped_entries():
    table = np.arange(12, dtype=np.float32).reshape(4, 3) + 1          # row 3 is the "dummy"
    indptr = np.array([0, 0, 2, 4], dtype=np.int64)                      # node 0 empty; 3 nodes; the table has 4 rows
    indices = np.array([1, 9, -1, 0], dtype=np.int32)                    # 9 and -1 read row 3
    mean = fn.csr_aggregate(table, indptr, indices, "mean")
    assert np.array_equal(mean[0], table[3])                             # empty row: the dummy row alone
    assert np.array_equal(mean[1], (np.float32(0) + table[1] + table[3]) / np.float32(2))
    assert np.array_equal(mean[3], table[3])                             # the dummy node n_nodes itself
    ms = fn.csr_aggregate(table, indptr, indices, "mean_self")
    assert np.array_equal(ms[0], (table[3] + table[0]) / np.float32(2))  # GCN divisor count + 1 over {N} U {v}
    assert np.array_equal(ms[3], (table[3] + table[3]) / np.float32(2))
    mx = fn.csr_aggregate(table, indptr, indices, "max", rows=np.array([2, -4], dtype=np.int32))
    assert np.array_equal(mx[0], np.maximum(table[3], table[0]))
    assert np.array_equal(mx[1], table[3])


def test_fixed_fanout_csr_equals_the_fanout_mean_bit_for_bit():
    rs = np.random.RandomState(5)
    n, k, F = 30, 7, 5
    table = rs.randn(50, F).astype(np.float32)
    ids = rs.randint(0, 50, size=n * k).astype(np.int32)
    indptr = np.arange(n + 1, dtype=np.int64) * k
    selfs = nu.gather_clamped(table, np.arange(n))
    rows = nu.gather_clamped(table, ids)
    assert nu.bits_equal(fn.csr_aggregate(table, indptr, ids, "mean", np.arange(n)), nu.mean_f32(rows, k))
    assert nu.bits_equal(fn.csr_aggregate(table, indptr, ids, "mean_self", np.arange(n)),
                         nu.mean_f32(rows, k, selfs, include_self=True))
    assert nu.bits_equal(fn.csr_aggregate(table, indptr, ids, "max", np.arange(n)), rows.reshape(n, k, F).max(axis=1))


def test_bf16_table_is_widened_exactly():
    rs = np.random.RandomState(6)
    bits = rs.randint(0, 2 ** 16, size=(20, 4)).astype(np.uint16)
    bits[(bits & 0x7F80) == 0x7F80] = 0                                  # no inf / NaN patterns
    indptr, indices = random_csr(rs, 15, 20, 6, bad=False)
    assert nu.bits_equal(fn.csr_aggregate(bits, indptr, indices, "mean"),
                         fn.csr_aggregate(nu.bf16_widen(bits), indptr, indices, "mean"))


# ---------------------------------------------------------------- neighbor_csr
@pytest.fixture(scope="module")
def toy_iterator():
    from test_walks_cpu import toy_graph
    G = toy_graph()
    id2idx = {n: i for i, n in enumerate(G.nodes())}
    return NodeMinibatchIterator(G, id2idx, None, {n: 0 for n in G.nodes()}, 1, batch_size=10, max_degree=25,
                                 rng=np.random.RandomState(0))


def unpadded_rows(c, train):
    rows = []
    for u in range(len(c["indptr"]) - 1):
        lo, hi = c["indptr"][u], c["indptr"][u + 1]
        nb = c["indices"][lo:hi]
        if train:
            nb = [] if c["val_or_test"][u] else nb[~c["edge_removed"][lo:hi]]
        rows.append(list(nb))
    return rows


@pytest.mark.parametrize("test", [False, True])
def test_neighbor_csr_keeps_the_rows_behind_the_padded_tables(toy_iterator, test):
    it = toy_iterator
    c = to_csr(it.G, it.id2idx)
    indptr, indices = it.neighbor_csr(test=test)
    assert indptr.dtype == np.int64 and indices.dtype == np.int32 and len(indptr) == len(it.id2idx) + 1
    got = [list(indices[indptr[u]:indptr[u + 1]]) for u in range(len(indptr) - 1)]
    assert got == unpadded_rows(c, train=not test)
    # every padded row draws from exactly these rows (construct_adj / construct_test_adj); empty rows stay all-N
    adj = it.test_adj if test else it.adj
    N = len(indptr) - 1
    for u in range(N):
        if got[u]:
            assert set(adj[u]) <= set(got[u])
        else:
            assert (adj[u] == N).all()
    if not test:
        assert indptr[-1] < len(c["indices"])                           # val/test rows and removed edges are gone


# ---------------------------------------------------------------- refusals (no GPU needed: they fire first)
def _bare_model(kind="mean"):
    """The attributes full_neighbor_embeddings reads before its first kernel launch."""
    m = SampleAndAggregate.__new__(SampleAndAggregate)
    m.aggregator_cls = {"mean": MeanAggregator, "seq": SeqAggregator}[kind]
    m.features = torch.zeros((5, 3))
    m.device = torch.device("cpu")
    m.aggregators = None
    return m


def test_refuses_the_seq_aggregator_and_sharded_tables():
    indptr, indices = np.zeros(5, np.int64), np.zeros(0, np.int32)
    with pytest.raises(NotImplementedError, match="seq"):
        _bare_model("seq").full_neighbor_embeddings(indptr, indices)
    m = _bare_model()
    m.features = type("Sharded", (), {"c_table": lambda self: None, "shape": (5, 3)})()
    with pytest.raises(NotImplementedError, match="ShardedFeatures"):
        m.full_neighbor_embeddings(indptr, indices)


def test_refuses_csr_of_the_wrong_dtype_length_or_device():
    m = _bare_model()
    with pytest.raises(TypeError, match="indptr"):
        m.full_neighbor_embeddings(np.zeros(5, np.int32), np.zeros(0, np.int32))
    with pytest.raises(TypeError, match="indices"):
        m.full_neighbor_embeddings(np.zeros(5, np.int64), np.zeros(0, np.int64))
    with pytest.raises(TypeError, match="indices"):
        m.full_neighbor_embeddings(torch.zeros(5, dtype=torch.int64), torch.zeros(0, dtype=torch.float32))
    with pytest.raises(ValueError, match="N \\+ 1"):
        m.full_neighbor_embeddings(np.zeros(4, np.int64), np.zeros(0, np.int32))
    m.device = torch.device("meta")
    with pytest.raises(ValueError, match="on cpu"):
        m.full_neighbor_embeddings(torch.zeros(5, dtype=torch.int64), torch.zeros(0, dtype=torch.int32))


def test_csr_aggregate_op_has_no_cpu_fallback():
    with pytest.raises(RuntimeError, match="CUDA-only"):
        ops.csr_aggregate(torch.zeros((3, 2)), torch.zeros(3, dtype=torch.int64), torch.zeros(0, dtype=torch.int32), "mean")
