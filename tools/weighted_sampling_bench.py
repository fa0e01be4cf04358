"""Time weighted neighbour sampling (sample_weight=) against the uniform draws on the GPU, alternating them in one process.

    python tools/weighted_sampling_bench.py [--iters 20] [--rounds 3] [--out weighted_sampling_bench.json]

Graphs, both built on the device by the R-MAT generator (synthetic.rmat_csr_device), with 602 random fp32 features and
41 classes:
  reddit     232,965 nodes, edge factor 490 (Reddit's node count and mean degree), a = 0.45, b = c = 0.22;
  powerlaw   2^20 nodes, edge factor 30, a = 0.57, b = c = 0.19: hub rows of 10^5 and more entries.
The sample weights are exp(2 z), z standard normal (a heavy-tailed spread over four orders of magnitude).  Each pair
below is timed uniform then weighted, --rounds times (CUDA events over --iters calls after a warm-up):
  blocks_ms      ops.csr_blocks for 512 random seeds with fanouts (25, 10), plan + size read + fill;
  step_ms        sampled_minibatch_train_step for the same seeds, mean aggregator, concat, width 128 per half, tf32x3.
keys: the number of keys the weighted blocks compute (the entries of the sampled rows of V_1 and V_2 with d > k, plan and
fill each), from the graph and one block set.  The card name, power limit and SM clock are read in the same command."""
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

F, C, B, FANOUTS = 602, 41, 512, [25, 10]


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


def graph(name):
    if name == "reddit":
        return rmat_csr_device(18, n_nodes=232965, edge_factor=490.0, a=0.45, b=0.22, c=0.22, d=0.11, seed=7)
    return rmat_csr_device(20, edge_factor=30.0, seed=7)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default="weighted_sampling_bench.json")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "the benchmark needs a CUDA device"
    gs._lib.lib()
    res = {"card": card(), "graphs": {}}
    g = torch.Generator(device="cuda").manual_seed(0)
    for name in ("reddit", "powerlaw"):
        indptr, indices = graph(name)
        n, nnz = indptr.numel() - 1, indices.numel()
        deg = torch.diff(indptr)
        sw = torch.exp(2 * torch.randn((nnz,), generator=g, device="cuda"))
        seeds = torch.randint(0, n, (B,), generator=g, device="cuda", dtype=torch.int32)
        # the keys of one block set's fill: rows of V_{l+1} longer than k_l
        blocks = ops.csr_blocks(indptr, indices, seeds, 2, fanouts=FANOUTS, seed=1, call=0, sample_weights=sw)
        keys = 0
        for l, k in enumerate(FANOUTS):
            nxt = blocks[l + 1].src_ids[:-1].long() if l + 1 < 2 else seeds.long().unique()
            d = deg.index_select(0, nxt.clamp(max=n - 1))
            keys += int(d[d > k].sum())
        info = {"nodes": n, "entries": nnz, "max_degree": int(deg.max()), "mean_degree": nnz / n,
                "keys_per_fill": keys}
        t = torch.zeros((n + 1, ops.pad_cols(F)), dtype=torch.float32, device="cuda")
        t[:-1, :F] = torch.randn((n, F), generator=g, device="cuda")
        adj = torch.zeros((n + 1, 1), dtype=torch.int32, device="cuda")
        gs.set_default_math("tf32x3")
        gs.inits.manual_seed(1)
        sampler = gs.UniformNeighborSampler(adj, seed=123)
        infos = [gs.SAGEInfo("node", sampler, FANOUTS[0], 128), gs.SAGEInfo("node", sampler, FANOUTS[1], 128)]
        m = gs.SupervisedGraphsage(C, {"batch_size": B, "dropout": 0.}, t[:, :F], adj, None, infos, concat=True,
                                   aggregator_type="mean", learning_rate=0.01)
        gs.set_default_math("fp32")
        labels = torch.zeros((B, C), device="cuda")
        labels[torch.arange(B, device="cuda"), torch.randint(0, C, (B,), generator=g, device="cuda")] = 1.0
        rounds = []
        for _ in range(a.rounds):
            rnd = {}
            for on in (False, True):
                kw = {"sample_weights": sw} if on else {}
                rnd["blocks_ms_" + ("weighted" if on else "uniform")] = timed(
                    lambda: ops.csr_blocks(indptr, indices, seeds, 2, fanouts=FANOUTS, seed=1, call=0, **kw), a.iters)
            for on in (False, True):
                kw = {"sample_weight": sw} if on else {}
                rnd["step_ms_" + ("weighted" if on else "uniform")] = timed(
                    lambda: m.sampled_minibatch_train_step(indptr, indices, seeds, labels, **kw), a.iters)
            print(json.dumps({name: rnd}), flush=True)
            rounds.append(rnd)
        info["rounds"] = rounds
        info["median"] = {k: float(np.median([r[k] for r in rounds])) for k in rounds[0]}
        res["graphs"][name] = info
        print(json.dumps({name: {k: v for k, v in info.items() if k != "rounds"}}), flush=True)
        del t, m, indptr, indices, sw, blocks
        torch.cuda.empty_cache()
    print(json.dumps({"card": res["card"]}))
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as fp:
        json.dump(res, fp, indent=1)


if __name__ == "__main__":
    main()
