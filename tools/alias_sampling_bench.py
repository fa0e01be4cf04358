"""Time the weighted fixed-fanout sampler (WeightedNeighborSampler, per-row alias tables) against the two uniform samplers
on the GPU, alternating them in one process.

    python tools/alias_sampling_bench.py [--iters 20] [--rounds 3] [--out alias_sampling_bench.json]

Graph: the Reddit-shaped R-MAT built on the device (synthetic.rmat_csr_device: 232,965 nodes, edge factor 490,
a = 0.45, b = c = 0.22), as tools/weighted_sampling_bench.py builds it, with weights exp(2 z), z standard normal, and 602
random fp32 features, 41 classes.  Reported:
  build_ms, table_bytes   ops.csr_alias_table once (set-up work), and the table's size;
  draw_ms_<sampler>       512 random seeds, fanouts (25, 10): sample_khop of UniformNeighborSampler (the padded table,
                          max_degree 128, built from the same CSR), two per-hop CSRNeighborSampler calls, and
                          WeightedNeighborSampler.sample_khop;
  step_ms_<sampler>       the graphed supervised graphsage_mean training step (concat, 128 per half, fp32) with each.
Each round times every variant in turn (CUDA events over --iters calls after an untimed one).  The card name, power
limit and SM clock are read in the same command."""
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
from graphsage_b200.synthetic import rmat_csr_device  # noqa: E402

F, C, B, FANOUTS, MAX_DEG = 602, 41, 512, [25, 10], 128


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def timed(fn, iters):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default="alias_sampling_bench.json")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "the benchmark needs a CUDA device"
    gs._lib.lib()
    g = torch.Generator(device="cuda").manual_seed(0)
    indptr, indices = rmat_csr_device(18, n_nodes=232965, edge_factor=490.0, a=0.45, b=0.22, c=0.22, d=0.11, seed=7)
    n, nnz = indptr.numel() - 1, indices.numel()
    w = torch.exp(2 * torch.randn((nnz,), generator=g, device="cuda"))
    res = {"card": card(), "nodes": n, "entries": nnz, "max_degree": int(torch.diff(indptr).max())}
    ops.csr_alias_table(indptr[:2].clone(), indices[:int(indptr[1])].clone(), w[:int(indptr[1])].clone())  # load
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    builds = []
    for _ in range(3):
        e0.record()
        table = ops.csr_alias_table(indptr, indices, w)
        e1.record()
        torch.cuda.synchronize()
        builds.append(e0.elapsed_time(e1))
        del table
    res["build_ms"] = builds
    adj, deg = ops.build_padded_adj(indptr, indices, MAX_DEG, seed=1)
    samplers = {"padded": gs.UniformNeighborSampler(adj, seed=123),
                "csr": gs.CSRNeighborSampler(indptr, indices, seed=123),
                "weighted": gs.WeightedNeighborSampler(indptr, indices, w, seed=123)}
    res["table_bytes"] = samplers["weighted"].table.numel() * 4
    seeds = torch.randint(0, n, (B,), generator=g, device="cuda", dtype=torch.int32)
    # fanouts in hop order: (10, 25) for samples_1 = 25, samples_2 = 10
    hop = [FANOUTS[1], FANOUTS[0]]

    def draws(s):
        if hasattr(s, "sample_khop"):
            return lambda: s.sample_khop(seeds, hop)

        def two():
            h1 = s((seeds, hop[0])).reshape(-1)
            return s((h1, hop[1]))
        return two

    t = torch.zeros((n + 1, ops.pad_cols(F)), dtype=torch.float32, device="cuda")
    t[:-1, :F] = torch.randn((n, F), generator=g, device="cuda")
    labels = torch.zeros((B, C), device="cuda")
    labels[torch.arange(B, device="cuda"), torch.randint(0, C, (B,), generator=g, device="cuda")] = 1.0
    steps = {}
    gs.set_default_math("fp32")
    for name, s in samplers.items():
        gs.inits.manual_seed(1)
        infos = [gs.SAGEInfo("node", s, FANOUTS[0], 128), gs.SAGEInfo("node", s, FANOUTS[1], 128)]
        m = gs.SupervisedGraphsage(C, {"batch_size": B, "dropout": 0.}, t[:, :F], adj, None, infos, concat=True,
                                   aggregator_type="mean", learning_rate=0.01)
        steps[name] = (m.graphed_train_step(B), m)
    rounds = []
    for _ in range(a.rounds):
        rnd = {}
        for name, s in samplers.items():
            rnd["draw_ms_" + name] = timed(draws(s), a.iters)
        for name, (step, _) in steps.items():
            rnd["step_ms_" + name] = timed(lambda: step(seeds, labels), a.iters)
        print(json.dumps(rnd), flush=True)
        rounds.append(rnd)
    res["rounds"] = rounds
    res["median"] = {k: float(np.median([r[k] for r in rounds])) for k in rounds[0]}
    res["spread"] = {k: float(max(r[k] for r in rounds) - min(r[k] for r in rounds)) for k in rounds[0]}
    print(json.dumps({k: v for k, v in res.items() if k != "rounds"}), flush=True)
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as fp:
        json.dump(res, fp, indent=1)


if __name__ == "__main__":
    main()
