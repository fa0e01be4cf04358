"""Time full-neighbourhood training with dropout (full_neighbor_train_step(dropout=p) and its minibatch form) on the
GPU, and the masked CSR kernels against the plain ones.

    python tools/full_neighbor_dropout_bench.py [--iters 5] [--rounds 2] [--out full_neighbor_dropout_bench.json]

Input: community_graph_csr(232,965, mean_deg=50) (Reddit's node count and density) with 602 random fp32 features and 41
classes, as tools/full_neighbor_train_bench.py; the train nodes are a fixed random 66 % of the nodes.  Model: 2 layers,
concat, width 128 per half, tf32x3 combine GEMMs, mean and max-pool.  Per aggregator and rate p in (0, 0.5):
  step_ms        full_neighbor_train_step(dropout=p) over every train node (CUDA events, --iters steps after a warm-up);
  peak_MB        torch.cuda.max_memory_allocated during those steps, above the resident set;
  mb_step_ms     full_neighbor_minibatch_train_step(dropout=p) for 512 seeds (the same seeds each step).
Kernels (layer 0, all N + 1 rows of the 602-wide table; CUDA events over --iters calls): csr_aggregate "mean" plain vs
masked, and the transposed "sum" plain vs masked (t_slot) on a 128-wide gradient.  Everything is measured --rounds times in
one process; the card name and power limit are read in the same command."""
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

F, C = 602, 41


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def timed(fn, iters):
    fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def build_model(kind, features, adj):
    gs.set_default_math("tf32x3")
    gs.inits.manual_seed(1)
    sampler = gs.UniformNeighborSampler(adj, seed=123)
    infos = [gs.SAGEInfo("node", sampler, 25, 128), gs.SAGEInfo("node", sampler, 10, 128)]
    m = gs.SupervisedGraphsage(C, {"batch_size": 512, "dropout": 0.}, features, adj, None, infos, concat=True,
                               aggregator_type=kind, learning_rate=0.01)
    gs.set_default_math("fp32")
    return m


def measure(kind, p, features, adj, indptr, indices, train, labels, seeds, seed_labels, iters):
    m = build_model(kind, features, adj)
    res = {"aggregator": kind, "rate": p}
    m.full_neighbor_train_step(indptr, indices, train, labels, dropout=p)          # warm-up: transposes cached
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    res["step_ms"] = timed(lambda: m.full_neighbor_train_step(indptr, indices, train, labels, dropout=p), iters)
    res["peak_MB"] = (torch.cuda.max_memory_allocated() - base) / 2**20
    res["mb_step_ms"] = timed(lambda: m.full_neighbor_minibatch_train_step(indptr, indices, seeds, seed_labels, dropout=p),
                              iters)
    return res


def kernels(features, indptr, indices, iters):
    n_rows = features.shape[0]
    pm = (indptr, None, indices.numel())
    site, self_site = (7, 1, 0.5), (7, 2, 0.5)
    res = {"mean_plain_ms": timed(lambda: ops.csr_aggregate(features, indptr, indices, "mean"), iters),
           "mean_masked_ms": timed(lambda: ops.csr_aggregate(features, indptr, indices, "mean",
                                                             dropout=(site, self_site, pm)), iters)}
    t_indptr, t_indices, t_slot = ops.csr_transpose(indptr, indices, slots=True)
    g = torch.randn((n_rows, 128), device="cuda")
    res["sum_plain_ms"] = timed(lambda: ops.csr_aggregate(g, t_indptr, t_indices, "sum"), iters)
    res["sum_masked_ms"] = timed(lambda: ops.csr_aggregate(g, t_indptr, t_indices, "sum", dropout=(site, self_site, pm),
                                                           t_slot=t_slot), iters)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--out", default="full_neighbor_dropout_bench.json")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "the benchmark needs a CUDA device"
    gs._lib.lib()
    res = {"card": card(), "rounds": []}
    ip, ix, _ = community_graph_csr(232965, mean_deg=50)
    n = len(ip) - 1
    res["graph"] = {"nodes": n, "entries": int(ip[-1]), "max_degree": int(np.diff(ip).max())}
    rs = np.random.RandomState(0)
    train = torch.from_numpy(np.sort(rs.choice(n, int(0.66 * n), replace=False)).astype(np.int32)).cuda()
    labels = torch.zeros((train.numel(), C), device="cuda")
    labels[torch.arange(train.numel(), device="cuda"), torch.from_numpy(rs.randint(0, C, train.numel())).cuda()] = 1.0
    seeds, seed_labels = train[:512], labels[:512]
    g = torch.Generator(device="cuda").manual_seed(0)
    t = torch.zeros((n + 1, ops.pad_cols(F)), dtype=torch.float32, device="cuda")
    t[:-1, :F] = torch.randn((n, F), generator=g, device="cuda")
    features = t[:, :F]
    adj = torch.from_numpy(padded_from_csr_fast(ip, ix, 128)[0]).cuda()
    indptr, indices = torch.from_numpy(ip).cuda(), torch.from_numpy(ix).cuda()
    for _ in range(a.rounds):
        rnd = [kernels(features, indptr, indices, a.iters)]
        rnd += [measure(kind, p, features, adj, indptr, indices, train, labels, seeds, seed_labels, a.iters)
                for kind in ("mean", "maxpool") for p in (0., 0.5)]
        for r in rnd:
            print(json.dumps(r), flush=True)
        res["rounds"].append(rnd)
    print(json.dumps({k: v for k, v in res.items() if k != "rounds"}))
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as fp:
        json.dump(res, fp, indent=1)


if __name__ == "__main__":
    main()
