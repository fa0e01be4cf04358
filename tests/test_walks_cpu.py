"""Random-walk co-occurrence pairs on the CPU: oracle/walks.py against the reference's own loop (tests/golden/walks.npz)
and against utils.run_random_walks driven by the contract's rng, chunking, the bounds and refusals, and the
`python -m graphsage_b200.utils` writer and its round trip through load_data."""
import os
import sys

import numpy as np
import pytest

from conftest import GOLDEN, load_golden

sys.path.insert(0, GOLDEN)
from make_walks_golden import hand_graph, toy_graph  # noqa: E402

from graphsage_b200 import utils  # noqa: E402
from graphsage_b200.graph import to_csr  # noqa: E402
from oracle import walks as ow  # noqa: E402


def index_space(G, nodes):
    pos = {n: i for i, n in enumerate(G.nodes())}
    csr = to_csr(G, pos)
    return csr["indptr"], csr["indices"], np.array([pos[n] for n in nodes], dtype=np.int32)


def cases():
    G = toy_graph()
    train = [n for n in G.nodes() if not G.node[n]["val"] and not G.node[n]["test"]]
    other = [n for n in G.nodes() if G.node[n]["val"] or G.node[n]["test"]]
    H, hand_nodes = hand_graph()
    return {"script": (G.subgraph(train), train, 50, 123, 0), "n2v": (G, other, 50, 123, 0),
            "hand": (H, hand_nodes, 3, 7, 5)}


CASES = cases()


def host_walks(G, nodes, num_walks, seed, counter):
    """utils.run_random_walks with the contract's rng: (node, context) names."""
    walked = [i for i, n in enumerate(nodes) if G.degree(n) > 0]
    rng = ow.ContractChoice(walked, num_walks, utils.WALK_LEN, seed, counter)
    pairs = utils.run_random_walks(G, nodes, num_walks=num_walks, rng=rng)
    assert rng.done()
    return pairs


@pytest.mark.parametrize("case", sorted(CASES))
def test_oracle_equals_the_reference_loop(case):
    G, nodes, W, seed, counter = CASES[case]
    got = ow.random_walks(*index_space(G, nodes), W, utils.WALK_LEN, seed, counter)
    want = load_golden("walks")[case + "_pairs"].astype(np.int32)
    assert got.dtype == np.int32 and got.shape == want.shape and np.array_equal(got, want)


def test_fixture_covers_the_hand_graph_edge_cases():
    d = load_golden("walks")
    G, nodes, *_ = CASES["hand"]
    assert list(d["hand_names"]) == G.nodes()
    pairs = d["hand_pairs"]
    names = G.nodes()
    assert G.degree("lone") == 0 and "lone" not in {names[a] for a, _ in pairs}
    assert all(a != b for a, b in pairs)                          # self co-occurrences (and the self loops) are dropped
    assert nodes.count("c") == 2 and ("c", "c") in [(u, v) for u, v in G.edges()]


@pytest.mark.parametrize("case", sorted(CASES))
def test_oracle_equals_the_host_loop_with_the_contract_rng(case):
    G, nodes, W, seed, counter = CASES[case]
    names = G.nodes()
    got = ow.random_walks(*index_space(G, nodes), W, utils.WALK_LEN, seed, counter)
    assert [(names[a], names[b]) for a, b in got.tolist()] == host_walks(G, nodes, W, seed, counter)


def test_draws_depend_on_seed_counter_and_position():
    base = ow.draws(123, 0, np.arange(4), 3, 9)
    assert base.shape == (4, 3, 8)
    for other in (ow.draws(124, 0, np.arange(4), 3, 9), ow.draws(123, 1, np.arange(4), 3, 9),
                  ow.draws(123, 0, np.arange(1, 5), 3, 9)):
        assert not np.array_equal(base, other)
    assert np.array_equal(ow.draws(123, 0, [2, 3], 3, 9), base[2:])


def test_chunks_with_their_start_offsets_give_one_call():
    G, nodes, W, seed, counter = CASES["n2v"]
    indptr, indices, starts = index_space(G, nodes)
    whole = ow.random_walks(indptr, indices, starts, W, 5, seed, counter)
    parts = [ow.random_walks(indptr, indices, starts[c:c + 37], W, 5, seed, counter, start_offset=c)
             for c in range(0, len(starts), 37)]
    assert np.array_equal(np.concatenate(parts), whole)
    assert not np.array_equal(ow.random_walks(indptr, indices, starts[37:], W, 5, seed, counter), whole[len(parts[0]):])


def test_directed_sinks_and_out_of_range_ids_end_a_walk():
    # 0 -> 1 -> 2 (a sink), 3 -> 99 (out of range); start ids -1 and 7 are outside [0, 4)
    indptr = np.array([0, 1, 2, 2, 3], np.int64)
    indices = np.array([1, 2, 99], np.int32)
    got = ow.random_walks(indptr, indices, np.array([0, 3, 2, -1, 7, 1], np.int32), 2, 6, 1)
    assert got.tolist() == [[0, 1], [0, 2]] * 2 + [[3, 99]] * 2 + [[1, 2]] * 2


def test_walk_lengths_and_counts():
    indptr, indices, starts = index_space(*CASES["hand"][:2])
    for L in (2, 5, 6, 33):
        for W in (1, 4):
            got = ow.random_walks(indptr, indices, starts, W, L, 9)
            assert len(got) <= len(starts) * W * (L - 1)
    assert ow.random_walks(indptr, indices, starts[:0], 3, 5, 1).shape == (0, 2)


@pytest.mark.parametrize("W,L", [(0, 5), (ow.MAX_WALKS + 1, 5), (1, 1), (1, ow.MAX_LEN + 1)])
def test_oracle_refuses_out_of_bounds(W, L):
    with pytest.raises(ValueError):
        ow.random_walks(np.array([0, 1], np.int64), np.array([0], np.int32), np.array([0], np.int32), W, L, 1)


@pytest.mark.parametrize("n,W,L", [(1, 0, 5), (1, (1 << 20) + 1, 5), (1, 1, 1), (1, 1, 34), (-1, 1, 5),
                                   (1 << 12, 1 << 20, 5)])
def test_library_refuses_out_of_bounds(built_lib, n, W, L):
    from graphsage_b200 import _lib
    assert _lib.lib().gs_random_walks_workspace_bytes(n, W, L) == -1
    assert b"gs_random_walks_workspace_bytes" in _lib.lib().gs_last_error_string()
    assert _lib.lib().gs_random_walks(None, None, 1, None, n, W, L, 0, 0, 0, None, 0, None, None) == -1
    assert _lib.lib().gs_random_walks_emit(None, n, W, L, None, 0, None, None) == -1


def test_library_bounds_match_the_oracle_and_the_binding(built_lib):
    from graphsage_b200 import _lib
    header = open(os.path.join(os.path.dirname(GOLDEN), "..", "include", "graphsage_b200.h")).read()
    assert "#define GS_WALK_MAX_WALKS (1 << 20)" in header and "#define GS_WALK_MAX_LEN 33" in header
    assert (_lib.WALK_MAX_WALKS, _lib.WALK_MAX_LEN) == (ow.MAX_WALKS, ow.MAX_LEN)
    assert "0x50000000" in header and ow.STREAM_WALK == 0x50000000


def test_random_walks_op_has_no_cpu_fallback():
    import torch
    from graphsage_b200 import ops
    with pytest.raises(RuntimeError):
        ops.random_walks(torch.zeros(2, dtype=torch.int64), torch.zeros(1, dtype=torch.int32),
                         torch.zeros(1, dtype=torch.int32), 1, 5, 1)


def _write_toy_dataset(prefix):
    G = toy_graph().subgraph(toy_graph().nodes()[:300])
    ids = G.nodes()
    utils.write_dataset(prefix, G, None, {n: i for i, n in enumerate(ids)}, {n: 0 for n in ids})
    return G


def test_main_writes_the_reference_text_for_the_train_subgraph(tmp_path):
    prefix = str(tmp_path / "toy")
    G = _write_toy_dataset(prefix)
    train = [n for n in G.nodes() if not G.node[n]["val"] and not G.node[n]["test"]]
    seen = {}

    def walker(H, nodes):
        seen.update(nodes=nodes, H=H)
        return host_walks(H, nodes, 4, 11, 0)

    out = str(tmp_path / "toy-walks.txt")
    pairs = utils.main([prefix + "-G.json", out], walker=walker)
    assert seen["nodes"] == train and seen["H"].nodes() == train
    assert sorted(seen["H"].edges()) == sorted((u, v) for u, v in G.subgraph(train).edges())
    text = open(out, "rb").read()
    assert text == "\n".join([str(p[0]) + "\t" + str(p[1]) for p in pairs]).encode()
    assert len(pairs) > 0 and not text.endswith(b"\n")
    walks = utils.load_data(prefix, load_walks=True)[3]
    assert walks == pairs


def test_main_keeps_string_ids_and_writes_nothing_for_no_pairs(tmp_path):
    import json
    g = {"directed": False, "multigraph": False, "graph": {},
         "nodes": [{"id": "x", "val": False, "test": False}, {"id": "y", "val": True, "test": False}],
         "links": [{"source": 0, "target": 1}]}
    path = str(tmp_path / "s-G.json")
    with open(path, "w") as fp:
        json.dump(g, fp)
    out = str(tmp_path / "s-walks.txt")
    assert utils.main([path, out], walker=lambda H, nodes: host_walks(H, nodes, 2, 1, 0)) == []
    assert open(out, "rb").read() == b""
    assert utils.format_walks([("x", "z"), ("q", 3)]) == "x\tz\nq\t3"


def test_main_takes_two_arguments():
    with pytest.raises(SystemExit):
        utils.main(["only-one"])


@pytest.fixture(scope="module")
def built_lib():
    from graphsage_b200.build import build_library
    return build_library()


def test_oracle_runs_reddit_sized_inputs_in_seconds():
    import time
    from graphsage_b200.synthetic import community_graph_csr
    indptr, indices, _ = community_graph_csr(50000, mean_deg=50, seed=5)
    starts = np.arange(0, 50000, 2, dtype=np.int32)
    t0 = time.time()
    got = ow.random_walks(indptr, indices, starts, 50, 5, 123)
    assert time.time() - t0 < 30
    assert 0.8 * len(starts) * 50 * 4 < len(got) <= len(starts) * 50 * 4
