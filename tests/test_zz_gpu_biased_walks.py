"""GPU: node2vec's biased walk (gs_random_walks_biased through ops.random_walks(p=, q=)) bit for bit against
oracle/biased_walks.py on toy-ppi, a community graph with hubs and a directed CSR with sinks, self loops, duplicates and
out-of-range ids; odd starts, walk lengths, seeds, counters, chunking and repeat runs; p == q == 1 against the uniform
walk; the transition law over about 10^6 walks; gs_csr_sort_rows against np.sort; run_random_walks_device(p, q); and a
Reddit-shaped call in WALK_CHUNK chunks."""
import numpy as np
import pytest
import torch

from oracle import biased_walks as bw
from test_biased_walks_cpu import check_frequencies, twelve_node_graph
from test_walks_cpu import CASES, index_space

pytestmark = pytest.mark.gpu

PQ = [(0.25, 4), (4, 0.25), (1e-4, 1e4)]


def cuda(a, dt):
    return torch.as_tensor(np.asarray(a), dtype=dt).cuda()


def device_walks(indptr, indices, starts, W, L, p, q, seed, counter=0, start_offset=0, sorted_indices=None):
    from graphsage_b200 import ops
    out = ops.random_walks(cuda(indptr, torch.int64), cuda(indices, torch.int32), cuda(starts, torch.int32), W, L, seed,
                           counter, start_offset, p=p, q=q, sorted_indices=sorted_indices)
    assert out.dtype == torch.int32 and out.is_cuda and out.dim() == 2 and out.shape[1] == 2
    return out.cpu().numpy()


def check(indptr, indices, starts, W, L, p, q, seed, counter=0, start_offset=0):
    got = device_walks(indptr, indices, starts, W, L, p, q, seed, counter, start_offset)
    want = bw.biased_random_walks(indptr, indices, starts, W, L, p, q, seed, counter, start_offset)
    assert got.shape == want.shape and np.array_equal(got, want), (got.shape, want.shape)
    return got


# ---- gs_csr_sort_rows ----------------------------------------------------------------------------------------------

def sort_rows(indptr, indices):
    from graphsage_b200 import ops
    return ops.csr_sort_rows(cuda(indptr, torch.int64), cuda(indices, torch.int32)).cpu().numpy()


def test_sort_rows_equals_np_sort_per_row():
    rs = np.random.RandomState(0)
    deg = rs.randint(0, 40, size=5000)
    deg[rs.random_sample(5000) < 0.2] = 0                               # empty rows
    deg[17], deg[4000], deg[4001] = 100000, 1, 300                      # a 10^5-entry row, a single entry, a medium row
    indptr = np.concatenate([[0], np.cumsum(deg)]).astype(np.int64)
    indices = rs.randint(-5, 6000, size=int(indptr[-1])).astype(np.int32)
    indices[rs.random_sample(len(indices)) < 0.01] = 2 ** 31 - 1
    got = sort_rows(indptr, indices)
    for i in range(len(deg)):
        a, b = indptr[i], indptr[i + 1]
        if b > a:
            assert np.array_equal(got[a:b], np.sort(indices[a:b])), i


def test_sort_rows_edge_cases():
    assert sort_rows(np.zeros(4, np.int64), np.zeros(0, np.int32)).shape == (0,)                 # E = 0
    assert sort_rows(np.zeros(1, np.int64), np.zeros(0, np.int32)).shape == (0,)                 # no nodes
    # rows cover [1, 5) only: the entries outside every row keep their values
    got = sort_rows(np.array([1, 3, 3, 5], np.int64), np.array([9, 4, 2, 8, 7, 6], np.int32))
    assert got.tolist() == [9, 2, 4, 7, 8, 6]


# ---- the biased walk against the oracle ----------------------------------------------------------------------------

@pytest.mark.parametrize("p,q", PQ)
@pytest.mark.parametrize("case", sorted(CASES))
def test_toy_cases_equal_the_oracle(case, p, q):
    G, nodes, W, seed, counter = CASES[case]
    check(*index_space(G, nodes), W, 5, p, q, seed, counter)


def community():
    from graphsage_b200.synthetic import community_graph_csr
    indptr, indices, _ = community_graph_csr(20000, mean_deg=30, seed=9)
    return indptr, indices


@pytest.mark.parametrize("p,q", PQ)
@pytest.mark.parametrize("W,L", [(50, 2), (50, 5), (3, 33)])
def test_community_graph_with_hubs(W, L, p, q):
    indptr, indices = community()
    deg = np.diff(indptr)
    assert deg.max() > 10 * deg.mean()
    starts = np.random.RandomState(W * 100 + L).randint(0, len(deg), size=1500).astype(np.int32)
    starts[:50] = np.argsort(deg)[-50:]
    check(indptr, indices, starts, W, L, p, q, 123)


def directed_csr():
    """Sinks, self loops, duplicates and out-of-range ids, rows in no particular order."""
    rs = np.random.RandomState(4)
    n = 3000
    deg = rs.randint(0, 9, size=n)
    indptr = np.concatenate([[0], np.cumsum(deg)]).astype(np.int64)
    indices = rs.randint(0, n, size=int(indptr[-1])).astype(np.int32)
    loops = rs.random_sample(len(indices)) < 0.05
    indices[loops] = np.repeat(np.arange(n), deg)[loops]               # self loops
    dup = np.flatnonzero((rs.random_sample(len(indices)) < 0.1) & (np.repeat(deg, deg) > 1))
    first = np.repeat(indptr[:-1], deg)[dup]
    indices[dup] = indices[first]                                       # duplicates of the row's first entry
    bad = rs.random_sample(len(indices)) < 0.03
    indices[bad] = rs.choice([-1, n, n + 7, 2 ** 31 - 1], size=int(bad.sum()))
    return indptr, indices


@pytest.mark.parametrize("p,q", PQ)
def test_directed_csr_with_sinks_loops_duplicates_and_out_of_range_ids(p, q):
    indptr, indices = directed_csr()
    n = len(indptr) - 1
    starts = np.random.RandomState(5).randint(0, n, size=2000).astype(np.int32)
    got = check(indptr, indices, starts, 20, 8, p, q, 77, counter=3)
    assert (got[:, 1] < 0).any() and (got[:, 1] >= n).any()


def test_odd_starts():
    indptr, indices = community()
    iso_indptr = np.concatenate([indptr, [indptr[-1]] * 3])
    n = len(iso_indptr) - 1
    starts = np.array([5, n - 1, -1, n, n + 100, 5, 5, n - 2, 17, -2 ** 31], np.int32)
    for p, q in PQ:
        check(iso_indptr, indices, starts, 50, 5, p, q, 1)
        assert device_walks(iso_indptr, indices, np.zeros(0, np.int32), 50, 5, p, q, 1).shape == (0, 2)
        assert device_walks(iso_indptr, indices, np.array([n - 1, -1], np.int32), 4, 5, p, q, 1).shape == (0, 2)


def test_fallback_is_exercised_and_exact():
    indptr, indices = community()
    starts = np.arange(0, 20000, 10, dtype=np.int32)
    pairs, stats = bw.biased_random_walks(indptr, indices, starts, 10, 5, 1e-4, 1e4, 3, stats=True)
    assert stats["fallbacks"] > 0.3 * stats["steps"]
    assert np.array_equal(device_walks(indptr, indices, starts, 10, 5, 1e-4, 1e4, 3), pairs)


def test_seeds_and_counters():
    indptr, indices = community()
    starts = np.arange(0, 2000, dtype=np.int32)
    outs = [check(indptr, indices, starts, 10, 5, 0.25, 4, seed, counter) for seed in (123, 124)
            for counter in (0, 1 << 33)]
    for a in range(4):
        for b in range(a + 1, 4):
            assert not np.array_equal(outs[a], outs[b])


def test_refusals():
    from graphsage_b200 import ops
    ip = torch.tensor([0, 1], dtype=torch.int64, device="cuda")
    ix = torch.zeros(1, dtype=torch.int32, device="cuda")
    st = torch.zeros(1, dtype=torch.int32, device="cuda")
    for p, q in [(1e-5, 1), (1, float("inf")), (0, 1), (1, -1), (float("nan"), 1)]:
        with pytest.raises(ValueError):
            ops.random_walks(ip, ix, st, 1, 5, 1, p=p, q=q)
    with pytest.raises(TypeError):
        ops.random_walks(ip, ix, st, 1, 5, 1, p=0.5, q=2, sorted_indices=ix.long())
    with pytest.raises(ValueError):
        ops.random_walks(ip, ix, st, 1, 5, 1, p=0.5, q=2, sorted_indices=torch.zeros(2, dtype=torch.int32, device="cuda"))
    assert ops.random_walks(ip, ix, st, 1 << 20, 33, 1, p=0.5, q=2).shape == (0, 2)        # a self loop: no pairs


def test_p_q_one_is_the_uniform_walk():
    from graphsage_b200 import ops
    indptr, indices = community()
    starts = np.random.RandomState(7).randint(0, 20000, size=3000).astype(np.int32)
    ip, ix, st = cuda(indptr, torch.int64), cuda(indices, torch.int32), cuda(starts, torch.int32)
    uniform = ops.random_walks(ip, ix, st, 20, 5, 9, 4).cpu().numpy()
    assert np.array_equal(ops.random_walks(ip, ix, st, 20, 5, 9, 4, p=1, q=1.0).cpu().numpy(), uniform)
    assert np.array_equal(ops.random_walks(ip, ix, st, 20, 5, 9, 4, p=1, q=1, sorted_indices=ops.csr_sort_rows(ip, ix))
                          .cpu().numpy(), uniform)
    assert not np.array_equal(ops.random_walks(ip, ix, st, 20, 5, 9, 4, p=1, q=1.5).cpu().numpy(), uniform)


def test_two_runs_are_identical_and_chunks_equal_one_call():
    from graphsage_b200 import ops
    indptr, indices = community()
    starts = np.random.RandomState(2).randint(0, 20000, size=10000).astype(np.int32)
    srt = ops.csr_sort_rows(cuda(indptr, torch.int64), cuda(indices, torch.int32))
    one = device_walks(indptr, indices, starts, 20, 5, 0.25, 4, 5, 2)
    assert np.array_equal(one, device_walks(indptr, indices, starts, 20, 5, 0.25, 4, 5, 2, sorted_indices=srt))
    bounds = [0, 1, 999, 4096, 4097, 10000]
    parts = [device_walks(indptr, indices, starts[a:b], 20, 5, 0.25, 4, 5, 2, start_offset=a, sorted_indices=srt)
             for a, b in zip(bounds, bounds[1:])]
    assert np.array_equal(np.concatenate(parts), one)
    check(indptr, indices, starts[4097:4600], 20, 5, 0.25, 4, 5, 2, start_offset=4097 + (1 << 31))


@pytest.mark.parametrize("p,q", PQ)
def test_transition_frequencies_over_a_million_walks(p, q):
    """65,536 disjoint copies of a 12-node directed graph, one walk of L = 3 from each copy's start, 16 rounds: a walk's
    pairs are the run of its start id (consecutive walks start in different copies), (t, v) then (t, x) unless x == t."""
    ip12, ix12 = twelve_node_graph()
    copies = 1 << 16
    deg = np.diff(ip12)
    indptr = np.concatenate([[0], np.cumsum(np.tile(deg, copies))]).astype(np.int64)
    indices = (np.tile(ix12, copies) + np.repeat(np.arange(copies) * 12, len(ix12))).astype(np.int32)
    ok = [i for i in range(12) if i not in ix12[ip12[i]:ip12[i + 1]]]   # starts without self loops: v != t
    local = np.array(ok)[np.arange(copies) % len(ok)]
    starts = np.tile(np.arange(copies) * 12 + local, 16).astype(np.int32)
    pairs = device_walks(indptr, indices, starts, 1, 3, p, q, 31, 5)
    head = np.concatenate([[True], pairs[1:, 0] != pairs[:-1, 0]])
    runs = np.diff(np.append(np.flatnonzero(head), len(pairs)))
    assert len(runs) == len(starts) and set(runs.tolist()) <= {1, 2}
    first = np.flatnonzero(head)
    t, v = pairs[first, 0], pairs[first, 1]
    x = np.where(runs == 2, pairs[np.minimum(first + 1, len(pairs) - 1), 1], t)
    assert (v // 12 == t // 12).all() and (x // 12 == t // 12).all()
    assert check_frequencies(ip12, ix12, t % 12, v % 12, x % 12, p, q, min_n=1000) >= 15


@pytest.mark.parametrize("case", ["hand", "script"])
def test_run_random_walks_device_returns_named_pairs(case, monkeypatch):
    from graphsage_b200 import ops, utils
    G, nodes, W, seed, counter = CASES[case]
    monkeypatch.setattr(utils, "WALK_CHUNK", 7)
    sorts = []
    real = ops.csr_sort_rows
    monkeypatch.setattr(ops, "csr_sort_rows", lambda *a: sorts.append(1) or real(*a))
    got = utils.run_random_walks_device(G, nodes, num_walks=W, seed=seed, counter=counter, p=0.25, q=4)
    assert len(sorts) == 1                                              # once per call, not per chunk
    names = G.nodes()
    want = bw.biased_random_walks(*index_space(G, nodes), W, utils.WALK_LEN, 0.25, 4, seed, counter)
    assert got == [(names[a], names[b]) for a, b in want.tolist()]
    if case == "hand":
        assert all(isinstance(a, str) and isinstance(b, str) for a, b in got)
    assert utils.run_random_walks_device(G, nodes, num_walks=W, seed=seed, counter=counter) == \
        utils.run_random_walks_device(G, nodes, num_walks=W, seed=seed, counter=counter, p=1, q=1)


def test_reddit_shaped_graph_in_chunks():
    from graphsage_b200 import _lib, ops, utils
    from graphsage_b200.synthetic import community_graph_csr
    indptr, indices, _ = community_graph_csr(232965, mean_deg=50, seed=123)
    starts = np.random.RandomState(0).permutation(232965)[:152410].astype(np.int32)
    ip, ix = cuda(indptr, torch.int64), cuda(indices, torch.int32)
    srt = ops.csr_sort_rows(ip, ix)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    C, W, L = utils.WALK_CHUNK, 50, 5
    total, outs = 0, []
    for c0 in range(0, len(starts), C):
        out = ops.random_walks(ip, ix, cuda(starts[c0:c0 + C], torch.int32), W, L, 123, 0, start_offset=c0, p=0.25, q=4,
                               sorted_indices=srt)
        total += len(out)
        outs.append(out.cpu().numpy())
        del out
    bound = _lib.lib().gs_random_walks_workspace_bytes(C, W, L) + C * W * (L - 1) * 8 + C * 4
    assert torch.cuda.max_memory_allocated() - base <= bound + (8 << 20), (torch.cuda.max_memory_allocated() - base, bound)
    assert total > 152410 * W * 3
    head = bw.biased_random_walks(indptr, indices, starts[:1500], W, L, 0.25, 4, 123)
    assert np.array_equal(outs[0][:len(head)], head)
    k = len(starts) - 1500
    tail = bw.biased_random_walks(indptr, indices, starts[k:], W, L, 0.25, 4, 123, start_offset=k)
    assert np.array_equal(outs[-1][len(outs[-1]) - len(tail):], tail)
