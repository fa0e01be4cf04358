"""node2vec's biased (p, q) walk on the CPU: the oracle (oracle/biased_walks.py) against a scalar restatement of the
contract, hand-computed classes and thresholds, the fallback draw, its transition law over many walks, the argument
refusals of the oracle, ops and the library, and `python -m graphsage_b200.utils --p/--q` through the walker seam."""
import math
import os

import numpy as np
import pytest

from conftest import GOLDEN

from graphsage_b200 import utils
from oracle import biased_walks as bw
from oracle import walks as ow
from oracle.philox import mulhi32, philox4x32_10, split64

T32 = 1 << 32


@pytest.mark.parametrize("p,q,want", [
    (1, 1, (T32, T32, T32)),
    (0.25, 4, (T32, T32 >> 2, T32 >> 4)),
    (4, 0.25, (T32 >> 4, T32 >> 2, T32)),
    (1, 2, (T32, T32, T32 >> 1)),                     # ties: return and in share the maximum
    (2, 1, (T32 >> 1, T32, T32)),                     # in and out share it
    (3, 1, (1431655765, T32, T32)),                   # floor(2^32 / 3)
    (1e-4, 1e4, (T32, 429496, 42)),                   # the bounds: floor(1e-4 * 2^32), floor(1e-8 * 2^32)
    (1e4, 1e-4, (42, 429496, T32)),
])
def test_thresholds(p, q, want):
    assert bw.thresholds(p, q) == want
    assert min(bw.thresholds(p, q)) >= 1


@pytest.mark.parametrize("p,q", [(0, 1), (1, 0), (-1, 1), (1, -0.5), (float("nan"), 1), (1, float("nan")),
                                 (float("inf"), 1), (1, float("inf")), (1e-5, 1), (1, 1e4 * 1.0001), (2e4, 1)])
def test_argument_errors(p, q):
    from graphsage_b200 import ops
    with pytest.raises(ValueError):
        bw.thresholds(p, q)
    with pytest.raises(ValueError):
        ops.check_walk_bias(p, q)
    with pytest.raises(ValueError):
        bw.biased_random_walks([0, 1], [0], [0], 1, 5, p, q, 1)


# A hand graph (n = 5): t = 0 -> {1, 2, 3}; v = 1 -> [0, 2, 2, 1, 4, 7]; 2 is a sink reached by 0 -> 2 with no 2 -> 0;
# 3 -> [0]; 4 -> [1]; 7 is outside [0, 5).
HAND_INDPTR = np.array([0, 3, 9, 9, 10, 11], np.int64)
HAND_INDICES = np.array([1, 2, 3, 0, 2, 2, 1, 4, 7, 0, 1], np.int32)


def test_hand_classes():
    # from v = 1 reached from t = 0: return (0), in (2, 2: a duplicate counts twice; 1: the self loop, 0 -> 1 exists),
    # out (4: 1 -> 4 but not 0 -> 4; 7: out of range)
    thr = bw.thresholds(0.5, 2)                              # a = (2, 1, 0.5): (2^32, 2^31, 2^30)
    assert thr == (T32, T32 >> 1, T32 >> 2)
    got = bw.transition_probs(HAND_INDPTR, HAND_INDICES, 0, 1, 0.5, 2)
    assert np.array_equal(got, np.array([4, 2, 2, 2, 1, 1], np.float64) / 12)
    # from v = 1 reached from t = 4 (row {1}): 4 is the return, 1 (an entry of 4's row) is in, the rest are out
    got = bw.transition_probs(HAND_INDPTR, HAND_INDICES, 4, 1, 0.5, 2)
    assert np.array_equal(got, np.array([1, 1, 1, 2, 4, 1], np.float64) / 10)
    # from v = 0 reached from t = 3 (row {0}): 1, 2 are out and 3 the return
    assert np.array_equal(bw.transition_probs(HAND_INDPTR, HAND_INDICES, 3, 0, 4, 0.25),
                          np.array([16, 16, 1], np.float64) / 33)


def words(seed, counter, pos, w, s, call):
    ctr = np.array([*split64(counter), pos, bw.STREAM_WALK_BIASED + ((w * 32 + s) << 3) + call], np.uint32)
    return [int(x) for x in philox4x32_10(ctr, np.array(split64(seed), np.uint32))]


def scalar_walk(indptr, indices, start, pos, w, walk_len, p, q, seed, counter):
    """One walk of the contract, entry by entry with Python integers: (visited, fell back at each move)."""
    thr = bw.thresholds(p, q)
    n = len(indptr) - 1
    visited, fell = [], []
    curr, prev = int(start), None
    if not 0 <= curr < n:
        return visited, fell
    for s in range(walk_len - 1):
        if not 0 <= curr < n:
            break
        row = [int(x) for x in indices[indptr[curr]:indptr[curr + 1]]]
        if not row:
            break

        def cls(x):
            if x == prev:
                return thr[0]
            return thr[1] if x in [int(y) for y in indices[indptr[prev]:indptr[prev + 1]]] else thr[2]
        if s == 0:
            nxt, fb = row[int(mulhi32(words(seed, counter, pos, w, s, 0)[0], len(row)))], False
        else:
            nxt = None
            for a in range(bw.ATTEMPTS):
                r = words(seed, counter, pos, w, s, a // 2)
                x = row[int(mulhi32(r[2 * (a % 2)], len(row)))]
                if r[2 * (a % 2) + 1] < cls(x):
                    nxt = x
                    break
            fb = nxt is None
            if fb:                                            # direct enumeration of the entries' target intervals
                r = words(seed, counter, pos, w, s, 7)
                u = r[0] + (r[1] << 32)
                wts = [cls(x) for x in row]
                target = u * sum(wts) >> 64
                lo = 0
                for x, wt in zip(row, wts):
                    if lo <= target < lo + wt:
                        nxt = x
                        break
                    lo += wt
        visited.append(nxt)
        fell.append(fb)
        prev, curr = curr, nxt
    return visited, fell


def check_against_scalar(indptr, indices, starts, W, L, p, q, seed, counter=0, start_offset=0):
    visited, moved, stats = bw.walk_paths(indptr, indices, starts, W, L, p, q, seed, counter, start_offset)
    fallbacks = 0
    for t, start in enumerate(starts):
        for w in range(W):
            g = t * W + w
            want, fell = scalar_walk(indptr, indices, start, start_offset + t, w, L, p, q, seed, counter)
            assert moved[g].sum() == len(want) and not moved[g, len(want):].any()
            assert visited[g, :len(want)].tolist() == want, (t, w)
            fallbacks += sum(fell)
    assert stats["fallbacks"] == fallbacks
    return stats


@pytest.mark.parametrize("p,q", [(0.5, 2), (0.25, 4), (4, 0.25), (1e-4, 1e4), (1e4, 1e-4)])
def test_oracle_steps_equal_the_scalar_contract_on_the_hand_graph(p, q):
    starts = np.array([0, 1, 3, 4, 2, -1, 5, 0], np.int32)
    check_against_scalar(HAND_INDPTR, HAND_INDICES, starts, 40, 6, p, q, 11, counter=3, start_offset=7)


def test_fallback_picks_by_inverse_cdf():
    # p = 1e4, q = 1e-4: out accepts always, return and in almost never.  From v = 1 reached from 0 every entry of row 1
    # but 4 and 7 is return or in, and from the clique below no entry is out at all, so rejection runs out.
    n = 6
    rows = [[j for j in range(n) if j != i] for i in range(n)]
    indptr = np.concatenate([[0], np.cumsum([len(r) for r in rows])]).astype(np.int64)
    indices = np.concatenate(rows).astype(np.int32)
    stats = check_against_scalar(indptr, indices, np.arange(n, dtype=np.int32), 30, 5, 1e4, 1e-4, 5)
    assert stats["fallbacks"] > 0.9 * stats["steps"] and stats["attempts"] >= bw.ATTEMPTS * stats["fallbacks"]
    stats = check_against_scalar(HAND_INDPTR, HAND_INDICES, np.array([0, 3], np.int32), 200, 3, 1e4, 1e-4, 6)
    assert stats["fallbacks"] > 0


def test_p_q_one_is_the_uniform_walk_and_chunks_equal_one_call():
    from graphsage_b200.synthetic import community_graph_csr
    indptr, indices, _ = community_graph_csr(3000, mean_deg=12, seed=3)
    starts = np.random.RandomState(1).randint(0, 3000, size=500).astype(np.int32)
    assert np.array_equal(bw.biased_random_walks(indptr, indices, starts, 7, 6, 1, 1, 9, 2),
                          ow.random_walks(indptr, indices, starts, 7, 6, 9, 2))
    whole = bw.biased_random_walks(indptr, indices, starts, 7, 6, 0.25, 4, 9, 2)
    parts = [bw.biased_random_walks(indptr, indices, starts[c:c + 123], 7, 6, 0.25, 4, 9, 2, start_offset=c)
             for c in range(0, len(starts), 123)]
    assert np.array_equal(np.concatenate(parts), whole)
    assert not np.array_equal(whole, bw.biased_random_walks(indptr, indices, starts, 7, 6, 4, 0.25, 9, 2))
    assert (whole[:, 0] != whole[:, 1]).all()


def twelve_node_graph():
    """A directed 12-node CSR with duplicates and self loops; every node has an entry and every id is in range."""
    rs = np.random.RandomState(12)
    rows = []
    for i in range(12):
        r = list(rs.choice(12, size=rs.randint(2, 6), replace=False))
        r += [r[0]] if i % 3 == 0 else []                    # duplicates
        r += [i] if i % 4 == 1 else []                       # self loops
        rows.append(r)
    indptr = np.concatenate([[0], np.cumsum([len(r) for r in rows])]).astype(np.int64)
    return indptr, np.concatenate(rows).astype(np.int32)


def node_law(indptr, indices, t, v, p, q):
    """{node id: probability} of the move from v reached from t (duplicate entries summed)."""
    law = {}
    for x, pr in zip(indices[indptr[v]:indptr[v + 1]].tolist(), bw.transition_probs(indptr, indices, t, v, p, q)):
        law[x] = law.get(x, 0.0) + pr
    return law


def check_frequencies(indptr, indices, t, v, x, p, q, min_n=200):
    """Every (t, v) cell with at least min_n moves: each node's count within 5 sigma of n * P(x | t, v)."""
    cells = 0
    for (tt, vv) in sorted(set(zip(t.tolist(), v.tolist()))):
        sel = (t == tt) & (v == vv)
        n = int(sel.sum())
        if n < min_n:
            continue
        cells += 1
        law = node_law(indptr, indices, tt, vv, p, q)
        got = {k: int(c) for k, c in zip(*np.unique(x[sel], return_counts=True))}
        assert set(got) <= set(law), (tt, vv)
        for k, pr in law.items():
            sigma = math.sqrt(n * pr * (1 - pr))
            assert abs(got.get(k, 0) - n * pr) <= 5 * sigma + 1e-9, (tt, vv, k, got.get(k, 0), n * pr)
    return cells


@pytest.mark.parametrize("p,q", [(0.25, 4), (4, 0.25), (1e-4, 1e4)])
def test_oracle_transition_frequencies_follow_the_law(p, q):
    indptr, indices = twelve_node_graph()
    starts = np.arange(12, dtype=np.int32)
    visited, moved, _ = bw.walk_paths(indptr, indices, starts, 20000, 3, p, q, 123, 1)
    assert moved.all()
    t = np.repeat(starts.astype(np.int64), 20000)
    assert check_frequencies(indptr, indices, t, visited[:, 0], visited[:, 1], p, q) >= 30


def test_constants_match_the_header_and_the_binding():
    from graphsage_b200 import _lib
    header = open(os.path.join(os.path.dirname(GOLDEN), "..", "include", "graphsage_b200.h")).read()
    assert "#define GS_WALK_PQ_MIN 1e-4" in header and "#define GS_WALK_PQ_MAX 1e4" in header
    assert "#define GS_WALK_BIASED_ATTEMPTS 14" in header and bw.ATTEMPTS == 14
    assert "0x60000000 + ((w * 32 + s) << 3) + call" in header and bw.STREAM_WALK_BIASED == 0x60000000
    assert (_lib.WALK_PQ_MIN, _lib.WALK_PQ_MAX) == (bw.PQ_MIN, bw.PQ_MAX)
    # the stream's span: the largest word is below 0x70000000
    assert bw.STREAM_WALK_BIASED + (((ow.MAX_WALKS - 1) * 32 + ow.MAX_LEN - 2) << 3) + 7 == 0x70000000 - 1


@pytest.fixture(scope="module")
def built_lib():
    from graphsage_b200.build import build_library
    return build_library()


@pytest.mark.parametrize("p,q", [(1e-5, 1), (1, float("inf")), (float("nan"), 1), (0, 1)])
def test_library_refuses_p_q(built_lib, p, q):
    from graphsage_b200 import _lib
    lib = _lib.lib()
    assert lib.gs_random_walks_biased(None, None, None, 1, None, 1, 1, 5, p, q, 0, 0, 0, None, 0, None, None) == -1
    assert b"gs_random_walks_biased" in lib.gs_last_error_string()


def test_library_refuses_sort_limits(built_lib):
    from graphsage_b200 import _lib
    lib = _lib.lib()
    for n_nodes, nnz in [(-1, 0), (0, -1), (1 << 31, 1), (1, 1 << 31)]:
        assert lib.gs_csr_sort_rows_workspace_bytes(n_nodes, nnz) == -1
        assert b"gs_csr_sort_rows_workspace_bytes" in lib.gs_last_error_string()
    assert lib.gs_csr_sort_rows_workspace_bytes(0, 0) == 0 and lib.gs_csr_sort_rows_workspace_bytes(5, 0) == 0
    assert lib.gs_csr_sort_rows(None, None, 5, 0, None, None, 0, None) == 0          # nothing to sort
    assert lib.gs_random_walks_biased(None, None, None, 1, None, 1, 0, 5, 0.5, 2, 0, 0, 0, None, 0, None, None) == -1


def test_ops_have_no_cpu_fallback():
    import torch
    from graphsage_b200 import ops
    ip, ix, st = torch.zeros(2, dtype=torch.int64), torch.zeros(1, dtype=torch.int32), torch.zeros(1, dtype=torch.int32)
    with pytest.raises(RuntimeError):
        ops.csr_sort_rows(ip, ix)
    with pytest.raises(RuntimeError):
        ops.random_walks(ip, ix, st, 1, 5, 1, p=0.5, q=2)
    with pytest.raises(ValueError):
        ops.random_walks(ip, ix, st, 1, 5, 1, p=0, q=2)


def _write_graph(tmp_path):
    import json
    g = {"directed": False, "multigraph": False, "graph": {},
         "nodes": [{"id": k, "val": k == 3, "test": False} for k in range(4)],
         "links": [{"source": 0, "target": 1}, {"source": 1, "target": 2}, {"source": 2, "target": 3}]}
    path = str(tmp_path / "g-G.json")
    with open(path, "w") as fp:
        json.dump(g, fp)
    return path


def test_main_without_p_q_calls_the_walker_as_before(tmp_path):
    path, out = _write_graph(tmp_path), str(tmp_path / "w.txt")
    seen = []

    def walker(H, nodes):                                     # exactly two parameters: no p, q passed
        seen.append(nodes)
        return [(0, 1), (1, 2)]
    assert utils.main([path, out], walker=walker) == [(0, 1), (1, 2)]
    assert seen == [[0, 1, 2]] and open(out, "rb").read() == b"0\t1\n1\t2"


@pytest.mark.parametrize("args,want", [(["--p", "0.25", "--q", "4"], (0.25, 4.0)), (["--q=0.5"], (1.0, 0.5)),
                                       (["--p", "2"], (2.0, 1.0)), (["--p", "1", "--q", "1"], (1.0, 1.0))])
def test_main_passes_p_q_to_the_walker(tmp_path, args, want):
    path, out = _write_graph(tmp_path), str(tmp_path / "w.txt")
    seen = []

    def walker(H, nodes, p, q):
        seen.append((p, q))
        return [(2, 0)]
    assert utils.main([path] + args + [out], walker=walker) == [(2, 0)]
    assert seen == [want] and open(out, "rb").read() == b"2\t0"


@pytest.mark.parametrize("argv", [["only-one"], ["a", "b", "c"], ["a", "b", "--p"], ["a", "b", "--p", "x"],
                                  ["a", "b", "--p", "0"], ["a", "b", "--q", "inf"], ["a", "b", "--q", "nan"],
                                  ["a", "--p", "0.5"]])
def test_main_usage_errors(argv):
    with pytest.raises(SystemExit) as e:
        utils.main(argv, walker=lambda *a, **k: [])
    assert "usage: python -m graphsage_b200.utils" in str(e.value)
