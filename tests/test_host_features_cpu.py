"""CPU: the host-memory feature table (graphsage_b200.HostFeatures) - argument checks, the hot-row choice, the staging
oracle (oracle/host_stage.py) on hand-made lists, and the refusals that need no device."""
import numpy as np
import pytest
import torch

from oracle import host_stage


def _table(n=10, F=5, dtype=np.float32, seed=0):
    t = np.random.RandomState(seed).randn(n + 1, F).astype(dtype)
    t[n] = 0
    return t


# ------------------------------------------------------------------ argument validation
@pytest.mark.parametrize("bad,err,match", [
    (np.zeros((4,), np.float32), ValueError, "2-D"),
    (np.zeros((4, 0), np.float32), ValueError, "2-D"),
    (np.zeros((4, 3), np.float64), TypeError, "float32 or bfloat16"),
    (np.zeros((4, 3), np.int32), TypeError, "float32 or bfloat16"),
    (np.ones((4, 3), np.float32), ValueError, "dummy row"),
])
def test_table_validation(bad, err, match):
    from graphsage_b200 import HostFeatures
    with pytest.raises(err, match=match):
        HostFeatures(bad)


@pytest.mark.parametrize("ids", [[3, 2], [1, 1], [-1, 2], [0, 10], [[1, 2]], [0.5]])
def test_cache_ids_validation(ids):
    from graphsage_b200 import HostFeatures
    with pytest.raises(ValueError, match="cache_ids"):
        HostFeatures(_table(), cache_ids=np.asarray(ids))


def test_registration_without_cuda_raises_the_library_error():
    from graphsage_b200 import HostFeatures
    if torch.cuda.is_available():
        pytest.skip("needs a CPU-only machine")
    with pytest.raises(RuntimeError, match="libgraphsage_b200 error"):
        HostFeatures(_table(), cache_ids=[0, 3, 9])
    with pytest.raises(RuntimeError, match="libgraphsage_b200 error"):
        HostFeatures(torch.from_numpy(_table(dtype=np.float32)).to(torch.bfloat16))


# ------------------------------------------------------------------ hot_rows
def _padded(rs, n, md):
    adj = rs.randint(0, n, size=(n + 1, md)).astype(np.int32)
    adj[:n][rs.rand(n) < 0.2] = n                 # some nodes have no neighbours (the dummy id)
    adj[n] = n
    return adj


def _brute_expected_reads(adj):
    """Per seed u uniform over [0, N): a hop-1 draw is a uniform entry of adj[u]; a hop-2 draw a uniform entry of the hop-1
    node's row.  Score = 10 P(hop 1 = v) + 250 P(hop 2 = v), summed entry by entry."""
    n, md = adj.shape[0] - 1, adj.shape[1]
    p1 = np.zeros(n + 1)
    for u in range(n):
        for v in adj[u]:
            p1[v] += 1.0
    p1 /= p1.sum()
    p2 = np.zeros(n + 1)
    for w in range(n):
        for v in adj[w]:
            p2[v] += p1[w] / md
    return (10 * p1 + 250 * p2)[:n]


def _is_top(score, chosen, n_rows):
    chosen = np.asarray(chosen)
    assert np.all(np.diff(chosen) > 0) and chosen.dtype == np.int64
    assert len(chosen) == min(n_rows, int((score > 0).sum()))
    rest = np.setdiff1d(np.arange(len(score)), chosen)
    if len(chosen) and len(rest):
        assert score[chosen].min() >= score[rest].max() - 1e-12
    assert (score[chosen] > 0).all()


@pytest.mark.parametrize("n_rows", [0, 1, 17, 60, 1000])
def test_hot_rows_padded_against_brute_force(n_rows):
    from graphsage_b200.host_features import hot_rows
    adj = _padded(np.random.RandomState(1), 120, 7)
    score = _brute_expected_reads(adj)
    got = hot_rows(adj, n_rows)
    _is_top(score, got, n_rows)
    assert np.array_equal(got, hot_rows(torch.from_numpy(adj), n_rows))


@pytest.mark.parametrize("n_rows", [0, 1, 25, 500])
def test_hot_rows_csr_against_brute_force(n_rows):
    from graphsage_b200.host_features import hot_rows
    rs = np.random.RandomState(2)
    n = 90
    deg = rs.randint(0, 6, size=n)
    indptr = np.concatenate([[0], np.cumsum(deg)]).astype(np.int64)
    indices = (rs.zipf(1.6, size=int(indptr[-1])) % n).astype(np.int32)
    cnt = np.zeros(n)
    for v in indices:
        cnt[v] += 1
    got = hot_rows((indptr, indices), n_rows)
    _is_top(cnt, got, n_rows)


def test_hot_remote_rows_unchanged_by_the_shared_score():
    """parallel.hot_remote_rows / hot_remote_rows_csr keep their choice: excluded own rows, the same top set."""
    from graphsage_b200 import parallel
    adj = _padded(np.random.RandomState(3), 200, 9)
    n = 200
    for world, rank in ((2, 0), (2, 1), (4, 3)):
        rs_ = parallel.uniform_bounds(n, world)
        lo, hi = rs_[rank], rs_[rank + 1]
        got = parallel.hot_remote_rows(adj, n, world, rank, 30)
        p1 = np.bincount(adj[lo:hi].reshape(-1), minlength=n + 1).astype(np.float64)
        p1 /= p1.sum()
        p2 = np.zeros(n + 1)
        for w in np.nonzero(p1[:n])[0]:
            np.add.at(p2, adj[w], p1[w] / adj.shape[1])
        score = (10 * p1 + 250 * p2)[:n]
        score[lo:hi] = -1
        _is_top(score, got, 30)
        assert not ((got >= lo) & (got < hi)).any()
        idx = torch.from_numpy(adj[:n].reshape(-1).copy())
        got_csr = parallel.hot_remote_rows_csr(idx, n, world, rank, 30)
        cnt = np.bincount(np.clip(adj[:n].reshape(-1), 0, n - 1), minlength=n).astype(np.int64)
        cnt[lo:hi] = -1
        assert len(got_csr) == 30 and not ((got_csr >= lo) & (got_csr < hi)).any()
        assert cnt[got_csr].min() >= np.delete(cnt, got_csr).max()


# ------------------------------------------------------------------ the staging oracle on hand-made lists
def test_oracle_stages_distinct_misses_once():
    n = 10
    table = _table(n, 3)
    cache = [2, 7]
    lists = [np.array([1, 2, 1, 10, -3]), np.array([7, 4, 1, 12, 4, 4]), np.array([], dtype=np.int64), np.array([9, 2])]
    ws, tr, staged = host_stage.stage(table, lists, cache)
    assert staged.tolist() == [1, 4, 9]                                   # first sightings, each miss once, no hits
    C = len(cache)
    assert tr[0].tolist() == [C + 1, 0, C + 1, C, C]
    assert tr[1].tolist() == [1, C + 2, C + 1, C, C + 2, C + 2]
    assert tr[2].tolist() == []
    assert tr[3].tolist() == [C + 3, 0]
    assert ws.shape == (C + 1 + 3, 3) and not ws[C].any()
    for ids, rows in zip(lists, tr):
        assert np.array_equal(ws[rows], table[host_stage.clamp_ids(ids, n)])


def test_oracle_edge_cases():
    n = 6
    table = _table(n, 2, seed=4)
    ws, tr, staged = host_stage.stage(table, [np.arange(n)], np.arange(n))     # everything cached: nothing staged
    assert len(staged) == 0 and tr[0].tolist() == list(range(n))
    ws, tr, staged = host_stage.stage(table, [np.array([n, n, -1])], [])      # only invalid ids: the zero row
    assert len(staged) == 0 and tr[0].tolist() == [0, 0, 0] and not ws.any()
    lists = [np.array([5, 5, 5]), np.array([0, 5])]
    ws, tr, staged = host_stage.stage(table, lists, [])
    assert staged.tolist() == [5, 0] and tr[0].tolist() == [1, 1, 1] and tr[1].tolist() == [2, 1]


# ------------------------------------------------------------------ refusals that need no device
def _fake_host():
    """A HostFeatures without its device state (the refusals look at the type and the dtype only)."""
    from graphsage_b200 import HostFeatures
    h = HostFeatures.__new__(HostFeatures)
    h.shape, h.dtype, h._alias = (11, 4), torch.float32, None
    return h


def test_refusals_without_a_device():
    import graphsage_b200 as gs
    from graphsage_b200.full_neighbor_training import refuse_full_neighbor
    h = _fake_host()
    with pytest.raises(NotImplementedError, match="identity_dim > 0 .*host-memory"):
        gs.SampleAndAggregate({}, h, np.zeros((11, 3), np.int32), None, [], identity_dim=4)
    for cls, args in ((gs.SupervisedGraphsage, (3, {})), (gs.UnsupervisedGraphsage, ({},))):
        with pytest.raises(NotImplementedError, match="distributed=True with a host-memory"):
            cls(*args, h, None, np.ones(10), [], distributed=True)

    class M(object):
        features, aggregator_cls = h, gs.MeanAggregator
    for training in (False, True):
        with pytest.raises(NotImplementedError, match="full-neighbourhood .*host-memory"):
            refuse_full_neighbor(M(), training)

    class P(object):
        features = h
    with pytest.raises(NotImplementedError, match="PipelinedForward with a host-memory"):
        gs.models.PipelinedForward(P(), 8)


def test_dims_and_dtype_refusals_read_the_host_table():
    """SampleAndAggregate.dims, refuse_dropout_table and refuse_seq_table need no special case."""
    from graphsage_b200.aggregators import refuse_seq_table
    from graphsage_b200.supervised_models import refuse_dropout_table
    h = _fake_host()
    assert not hasattr(h, "c_table")
    refuse_dropout_table(h)
    refuse_seq_table(h)
    h.dtype = torch.bfloat16
    with pytest.raises(NotImplementedError, match="bfloat16 feature table"):
        refuse_dropout_table(h)
    with pytest.raises(NotImplementedError, match="bfloat16 feature table"):
        refuse_seq_table(h)
