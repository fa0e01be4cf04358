"""Time minibatch training over sampled blocks (SupervisedGraphsage.sampled_minibatch_train_step) on the GPU, against
the sampled tree path (train_step, graphed_train_step) and the whole-neighbourhood blocks on the same ids.

    python tools/sampled_blocks_bench.py [--iters 10] [--rounds 2] [--out sampled_blocks_bench.json] [--dropout P]

Graph: community_graph_csr(232,965, mean_deg=50) - Reddit's node count, hub-heavy - with 602 random fp32 features.
Model: 2 layers, concat, width 128 per half, tf32x3 combine GEMMs, 41 classes, layer_infos fanouts (25, 10) as the
reference's supervised_train sets them (hop 1 from the seeds uses layer_infos[1]); mean and max-pool; batches of 512
random node ids.  Per case, after one warm-up of each step:
  V, entries        |V_0|, |V_1| and the entries of blocks 0 and 1 of the sampled blocks (|V_2| is the batch);
  tree_rows         the rows the tree path gathers per hop: 512, 512 k_hop1, 512 k_hop1 k_hop2 (from the shapes);
  full_V, full_entries   the same for the whole-neighbourhood blocks;
  blocks_ms         one ops.csr_blocks(..., fanouts) call, its device-to-host read of the sizes included;
  full_blocks_ms    one whole-neighbourhood ops.csr_blocks call;
  step_ms           sampled_minibatch_train_step end to end (--iters steps, CUDA events), peak_MB above the resident set;
  tree_step_ms      train_step;  graphed_step_ms  graphed_train_step's replays;
  full_step_ms      full_neighbor_minibatch_train_step ("oom" if it does not fit).
With --dropout P only the sampled step is timed, at dropout=0 and dropout=P alternately (step_ms_p0, step_ms_p, and
their peak_MB), for the cost of the training masks (oracle/sampled_blocks_dropout.py) on this path.
Everything is measured --rounds times in one process; the card name and power limit are read in the same command."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import graphsage_b200 as gs  # noqa: E402
from graphsage_b200 import ops  # noqa: E402
from graphsage_b200.minibatch import padded_from_csr_fast  # noqa: E402
from graphsage_b200.synthetic import community_graph_csr  # noqa: E402

C, F, N_NODES, MEAN_DEG, BATCH, FANOUTS = 41, 602, 232965, 50, 512, (25, 10)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


class Timer(object):
    def __enter__(self):
        self.e0, self.e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        self.e0.record()
        return self

    def __exit__(self, *exc):
        self.e1.record()
        torch.cuda.synchronize()
        self.ms = self.e0.elapsed_time(self.e1)


def build_model(kind, features, adj):
    gs.set_default_math("tf32x3")
    gs.inits.manual_seed(1)
    sampler = gs.UniformNeighborSampler(adj, seed=123)
    infos = [gs.SAGEInfo("node", sampler, k, 128) for k in FANOUTS]
    m = gs.SupervisedGraphsage(C, {"batch_size": BATCH, "dropout": 0.}, features, adj, None, infos, concat=True,
                               aggregator_type=kind, learning_rate=0.01)
    gs.set_default_math("fp32")
    return m


def tree_rows(fanouts, batch):
    """Rows per hop of the tree path: hop h from the seeds uses layer_infos[L - h] (reference models.py:268-272)."""
    rows, n = [batch], batch
    for k in reversed(fanouts):
        n *= k
        rows.append(n)
    return rows


def timed_steps(step, iters):
    """(ms per step, peak MB above the resident set) of `iters` calls of step()."""
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    with Timer() as t:
        for _ in range(iters):
            step()
    return t.ms / iters, (torch.cuda.max_memory_allocated() - base) / 2**20


def measure(kind, features, adj, indptr, indices, ids, labels, iters):
    m = build_model(kind, features, adj)
    sampler = m.layer_infos[0].neigh_sampler
    res = {"aggregator": kind, "batch": int(ids.numel()), "fanouts": list(FANOUTS),
           "tree_rows": tree_rows(FANOUTS, int(ids.numel()))}
    blocks = ops.csr_blocks(indptr, indices, ids, 2, fanouts=FANOUTS, seed=sampler.seed, call=0)
    res["V"] = [int(b.src_ids.numel()) for b in blocks]
    res["entries"] = [int(b.indices.numel()) for b in blocks]
    del blocks
    with Timer() as t:
        ops.csr_blocks(indptr, indices, ids, 2, fanouts=FANOUTS, seed=sampler.seed, call=1)
    res["blocks_ms"] = t.ms
    full = ops.csr_blocks(indptr, indices, ids, 2)
    res["full_V"] = [int(b.src_ids.numel()) for b in full]
    res["full_entries"] = [int(b.indices.numel()) for b in full]
    del full
    with Timer() as t:
        ops.csr_blocks(indptr, indices, ids, 2)
    res["full_blocks_ms"] = t.ms
    m.sampled_minibatch_train_step(indptr, indices, ids, labels)                  # warm-up: Adam state
    res["step_ms"], res["peak_MB"] = timed_steps(lambda: m.sampled_minibatch_train_step(indptr, indices, ids, labels),
                                                 iters)
    host_ids = ids.cpu()
    m.train_step(host_ids, labels)
    res["tree_step_ms"], res["tree_peak_MB"] = timed_steps(lambda: m.train_step(host_ids, labels), iters)
    step = m.graphed_train_step(int(ids.numel()))
    step(ids, labels)
    res["graphed_step_ms"], _ = timed_steps(lambda: step(ids, labels), iters)
    del step
    torch.cuda.empty_cache()
    try:
        m.full_neighbor_minibatch_train_step(indptr, indices, ids, labels)
        res["full_step_ms"], res["full_peak_MB"] = timed_steps(
            lambda: m.full_neighbor_minibatch_train_step(indptr, indices, ids, labels), iters)
    except torch.cuda.OutOfMemoryError:
        res["full_step_ms"] = res["full_peak_MB"] = "oom"
    torch.cuda.empty_cache()
    return res


def measure_dropout(kind, features, adj, indptr, indices, ids, labels, iters, p):
    """sampled_minibatch_train_step at dropout 0 and p, alternating, after a warm-up of each."""
    m = build_model(kind, features, adj)
    res = {"aggregator": kind, "batch": int(ids.numel()), "fanouts": list(FANOUTS), "dropout": p}
    for rate in (0., p):
        m.sampled_minibatch_train_step(indptr, indices, ids, labels, dropout=rate)
    for rep in range(2):
        for rate, key in ((0., "p0"), (p, "p")):
            ms, mb = timed_steps(lambda: m.sampled_minibatch_train_step(indptr, indices, ids, labels, dropout=rate),
                                 iters)
            res.setdefault("step_ms_" + key, []).append(ms)
            res.setdefault("peak_MB_" + key, []).append(mb)
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--out", default="sampled_blocks_bench.json")
    ap.add_argument("--dropout", type=float, default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "the benchmark needs a CUDA device"
    gs._lib.lib()
    res = {"card": card(), "rounds": [[] for _ in range(a.rounds)]}
    print(json.dumps({"card": res["card"]}), flush=True)
    ip, ix, _ = community_graph_csr(N_NODES, mean_deg=MEAN_DEG)
    n = len(ip) - 1
    res["graph"] = {"nodes": n, "entries": int(ip[-1]), "max_degree": int(np.diff(ip).max()), "features": F}
    print(json.dumps(res["graph"]), flush=True)
    g = torch.Generator(device="cuda").manual_seed(0)
    t = torch.zeros((n + 1, ops.pad_cols(F)), dtype=torch.float32, device="cuda")
    t[:-1, :F] = torch.randn((n, F), generator=g, device="cuda")
    features = t[:, :F]
    adj = torch.from_numpy(padded_from_csr_fast(ip, ix, 128)[0]).cuda()
    indptr, indices = torch.from_numpy(ip).cuda(), torch.from_numpy(ix).cuda()
    rs = np.random.RandomState(0)
    for r in range(a.rounds):
        for kind in ("mean", "maxpool"):
            ids = torch.from_numpy(rs.choice(n, BATCH, replace=False).astype(np.int32)).cuda()
            labels = torch.zeros((BATCH, C), device="cuda")
            labels[torch.arange(BATCH, device="cuda"), torch.from_numpy(rs.randint(0, C, BATCH)).cuda()] = 1.0
            if a.dropout is not None:
                out = dict(round=r, **measure_dropout(kind, features, adj, indptr, indices, ids, labels, a.iters,
                                                      a.dropout))
            else:
                out = dict(round=r, **measure(kind, features, adj, indptr, indices, ids, labels, a.iters))
            print(json.dumps(out), flush=True)
            res["rounds"][r].append(out)
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as fp:
        json.dump(res, fp, indent=1)


if __name__ == "__main__":
    main()
