"""GPU: gs_random_walks / gs_random_walks_emit (ops.random_walks) bit for bit against oracle/walks.py on the toy-ppi
cases, a community graph with hubs, a directed CSR with sinks and out-of-range neighbour ids, odd starts, W / L / seed /
counter variations and a Reddit-shaped input; reproducibility and chunking; run_random_walks_device; and
`python -m graphsage_b200.utils` end to end, followed by a few unsupervised training steps on the file it wrote."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from conftest import ROOT
from oracle import walks as ow
from test_walks_cpu import CASES, host_walks, index_space
from test_zz_gpu_train_cli import toy  # noqa: F401  (fixture: the toy-ppi dataset with walks)

pytestmark = pytest.mark.gpu


def device_walks(indptr, indices, starts, W, L, seed, counter=0, start_offset=0):
    from graphsage_b200 import ops
    cuda = lambda a, dt: torch.as_tensor(np.asarray(a), dtype=dt).cuda()
    out = ops.random_walks(cuda(indptr, torch.int64), cuda(indices, torch.int32), cuda(starts, torch.int32), W, L, seed,
                           counter, start_offset)
    assert out.dtype == torch.int32 and out.is_cuda and out.dim() == 2 and out.shape[1] == 2
    return out.cpu().numpy()


def check(indptr, indices, starts, W, L, seed, counter=0, start_offset=0):
    got = device_walks(indptr, indices, starts, W, L, seed, counter, start_offset)
    want = ow.random_walks(indptr, indices, starts, W, L, seed, counter, start_offset)
    assert got.shape == want.shape and np.array_equal(got, want), (got.shape, want.shape)
    return got


@pytest.mark.parametrize("case", sorted(CASES))
def test_toy_cases_equal_the_oracle_and_the_fixture(case, golden):
    G, nodes, W, seed, counter = CASES[case]
    got = check(*index_space(G, nodes), W, 5, seed, counter)
    assert np.array_equal(got, golden("walks")[case + "_pairs"].astype(np.int32))


def community():
    from graphsage_b200.synthetic import community_graph_csr
    indptr, indices, _ = community_graph_csr(20000, mean_deg=30, seed=9)
    return indptr, indices


@pytest.mark.parametrize("W,L", [(1, 2), (1, 5), (50, 2), (50, 5), (3, 33), (7, 9)])
def test_community_graph_with_hubs(W, L):
    indptr, indices = community()
    deg = np.diff(indptr)
    assert deg.max() > 10 * deg.mean()                                  # hubs
    starts = np.random.RandomState(W * 100 + L).randint(0, len(deg), size=3000).astype(np.int32)
    starts[:50] = np.argsort(deg)[-50:]
    check(indptr, indices, starts, W, L, 123)


def test_directed_csr_with_sinks_and_out_of_range_neighbours():
    rs = np.random.RandomState(4)
    n = 3000
    deg = rs.randint(0, 6, size=n)                                      # about one row in six is a sink
    indptr = np.concatenate([[0], np.cumsum(deg)]).astype(np.int64)
    indices = rs.randint(0, n, size=int(indptr[-1])).astype(np.int32)
    bad = rs.random_sample(len(indices)) < 0.05
    indices[bad] = rs.choice([-1, n, n + 7, 2 ** 31 - 1], size=int(bad.sum()))
    starts = rs.randint(0, n, size=2000).astype(np.int32)
    got = check(indptr, indices, starts, 20, 8, 77, counter=3)
    assert (got[:, 1] < 0).any() and (got[:, 1] >= n).any()            # out-of-range ids are emitted, then the walk stops


def test_odd_starts():
    indptr, indices = community()
    iso_indptr = np.concatenate([indptr, [indptr[-1]] * 3])          # three extra nodes without neighbours
    n = len(iso_indptr) - 1
    starts = np.array([5, n - 1, -1, n, n + 100, 5, 5, n - 2, 17, -2 ** 31], np.int32)
    check(iso_indptr, indices, starts, 50, 5, 1)
    assert device_walks(iso_indptr, indices, np.zeros(0, np.int32), 50, 5, 1).shape == (0, 2)
    assert device_walks(iso_indptr, indices, np.array([n - 1, -1], np.int32), 4, 5, 1).shape == (0, 2)


def test_seeds_and_counters_give_different_walks():
    indptr, indices = community()
    starts = np.arange(0, 2000, dtype=np.int32)
    outs = [check(indptr, indices, starts, 10, 5, seed, counter) for seed in (123, 124) for counter in (0, 1 << 33)]
    for a in range(4):
        for b in range(a + 1, 4):
            assert not np.array_equal(outs[a], outs[b])


def test_two_calls_are_bit_identical_and_chunks_equal_one_call():
    indptr, indices = community()
    starts = np.random.RandomState(2).randint(0, 20000, size=10000).astype(np.int32)
    one = device_walks(indptr, indices, starts, 50, 5, 5, 2)
    assert np.array_equal(one, device_walks(indptr, indices, starts, 50, 5, 5, 2))
    bounds = [0, 1, 999, 4096, 4097, 10000]
    parts = [device_walks(indptr, indices, starts[a:b], 50, 5, 5, 2, start_offset=a) for a, b in zip(bounds, bounds[1:])]
    assert np.array_equal(np.concatenate(parts), one)
    check(indptr, indices, starts[4097:], 50, 5, 5, 2, start_offset=4097 + (1 << 31))


def test_reddit_shaped_graph():
    from graphsage_b200.synthetic import community_graph_csr
    indptr, indices, _ = community_graph_csr(232965, mean_deg=50, seed=123)
    starts = np.random.RandomState(0).permutation(232965)[:152410].astype(np.int32)
    got = check(indptr, indices, starts, 50, 5, 123)
    assert len(got) > 152410 * 50 * 3


def test_refusals():
    from graphsage_b200 import ops
    ip = torch.tensor([0, 1], dtype=torch.int64, device="cuda")
    ix = torch.zeros(1, dtype=torch.int32, device="cuda")
    st = torch.zeros(1, dtype=torch.int32, device="cuda")
    with pytest.raises(TypeError):
        ops.random_walks(ip.int(), ix, st, 1, 5, 1)
    with pytest.raises(TypeError):
        ops.random_walks(ip, ix.long(), st, 1, 5, 1)
    with pytest.raises(TypeError):
        ops.random_walks(ip, ix, st.long(), 1, 5, 1)
    for W, L in [(0, 5), ((1 << 20) + 1, 5), (1, 1), (1, 34)]:
        with pytest.raises(ValueError):
            ops.random_walks(ip, ix, st, W, L, 1)
    with pytest.raises(ValueError):
        ops.random_walks(ip, ix, st, 1, 5, 1, start_offset=2 ** 32)
    with pytest.raises(RuntimeError):
        ops.random_walks(ip, ix, st.cpu(), 1, 5, 1)
    assert ops.random_walks(ip, ix, st, 1 << 20, 33, 1).shape == (0, 2)           # the bounds themselves (a self loop)
    assert ops.random_walks(ip, ix, st, 1, 2, 1).shape == (0, 2)


@pytest.mark.parametrize("case", ["hand", "script"])
def test_run_random_walks_device_returns_named_pairs(case, monkeypatch):
    from graphsage_b200 import utils
    G, nodes, W, seed, counter = CASES[case]
    monkeypatch.setattr(utils, "WALK_CHUNK", 7)                         # many chunks
    got = utils.run_random_walks_device(G, nodes, num_walks=W, seed=seed, counter=counter)
    assert got == host_walks(G, nodes, W, seed, counter)
    if case == "hand":
        assert all(isinstance(a, str) and isinstance(b, str) for a, b in got)


def test_utils_entry_point_writes_the_walks_file_and_the_trainer_reads_it(toy, tmp_path):
    from graphsage_b200 import unsupervised_train as unsup, utils
    from graphsage_b200.graph import node_link_graph
    import json
    out = [str(tmp_path / ("walks%d.txt" % k)) for k in range(2)]
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    for path in out:
        r = subprocess.run([sys.executable, "-m", "graphsage_b200.utils", toy + "-G.json", path], cwd=ROOT, env=env,
                           capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stderr
    text = open(out[0], "rb").read()
    assert text == open(out[1], "rb").read()
    G = node_link_graph(json.load(open(toy + "-G.json")))
    nodes = [n for n in G.nodes() if not G.node[n]["val"] and not G.node[n]["test"]]
    H = G.subgraph(nodes)
    want = host_walks(H, nodes, utils.N_WALKS, 123, 0)
    assert text == "\n".join([str(p[0]) + "\t" + str(p[1]) for p in want]).encode()
    # the unsupervised trainer on that walks file
    os.replace(out[0], toy + "-walks.txt")
    data = utils.load_data(toy, load_walks=True)
    assert data[3] == want
    flags = unsup.parse_flags(["--train_prefix", toy, "--base_log_dir", str(tmp_path), "--model", "graphsage_mean",
                               "--dim_1", "16", "--dim_2", "16", "--batch_size", "128", "--max_total_steps", "6",
                               "--validate_iter", "3", "--validate_batch_size", "64", "--print_every", "3", "--epochs",
                               "1", "--gpu", "0"])
    m = unsup.train(data, flags, device=torch.device("cuda", 0))
    assert all(torch.isfinite(p).all() for p in m.parameters())
