"""Time the weighted CSR reductions (edge_weight=) against the unweighted ones on the GPU, alternating them in one process.

    python tools/weighted_csr_bench.py [--iters 10] [--rounds 3] [--out weighted_csr_bench.json]

Input: community_graph_csr(232,965, mean_deg=50) (Reddit's node count and density) with 602 random fp32 features and 41
classes, as tools/full_neighbor_train_bench.py; the train nodes are a fixed random 66 % of the nodes; the edge weights
are uniform in [0, 2).  Model: 2 layers, concat, width 128 per half, tf32x3 combine GEMMs.  Each pair below is timed
unweighted then weighted, --rounds times (CUDA events over --iters calls after a warm-up):
  mean_ms        csr_aggregate "mean" over layer 0's 602-wide table, all N + 1 rows (gs_csr_aggregate[_weighted]);
  sum_ms         the transposed "sum" on a 128-wide gradient (the backward of the means);
  max_bwd_ms     csr_max_backward on a 128-wide MLP output (both phases);
  step_ms        full_neighbor_train_step over every train node, mean and max-pool;
  sampled_ms     sampled_minibatch_train_step for 512 seeds with fanouts (25, 10), mean.
bytes: the algorithmic reads of the layer-0 mean (one 602-wide fp32 row per entry and per row, the CSR, and the weights),
against which the kernel time gives a rate.  The card name, power limit and SM clock are read in the same command."""
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


def pair(name, fn, iters):
    """{name_plain: ms, name_weighted: ms}: fn(False) (unweighted) then fn(True) (weighted).  timed() makes one untimed
    call first; the training-step pairs depend on it, since the model caches one FullNeighborGraph, keyed by the weight
    tensor too, so the first call after a switch rebuilds the transposes (and their weights) outside the timed window."""
    return {name + "_plain": timed(lambda: fn(False), iters), name + "_weighted": timed(lambda: fn(True), iters)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default="weighted_csr_bench.json")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "the benchmark needs a CUDA device"
    gs._lib.lib()
    res = {"card": card(), "rounds": []}
    ip, ix, _ = community_graph_csr(232965, mean_deg=50)
    n, nnz = len(ip) - 1, int(ip[-1])
    res["graph"] = {"nodes": n, "entries": nnz, "max_degree": int(np.diff(ip).max())}
    rows = n + 1 + nnz                       # rows read by the mean: one per entry, plus the dummy row of empty rows
    res["mean_bytes_plain"] = rows * F * 4 + (n + 1) * 8 + nnz * 4
    res["mean_bytes_weighted"] = res["mean_bytes_plain"] + nnz * 4
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
    w = torch.rand((nnz,), generator=g, device="cuda") * 2
    t_indptr, t_indices, t_slot = ops.csr_transpose(indptr, indices, slots=True)
    tw = ops.csr_transpose_weights(w, indptr, t_indices, t_slot)
    grad = torch.randn((n + 1, 128), generator=g, device="cuda")
    z = torch.relu(torch.randn((n + 1, 128), generator=g, device="cuda"))
    dm = torch.randn((n + 1, 128), generator=g, device="cuda")
    m_plain = ops.csr_aggregate(z, indptr, indices, "max").clone()
    m_weighted = ops.csr_aggregate(z, indptr, indices, "max", weights=w).clone()
    models = {kind: build_model(kind, features, adj) for kind in ("mean", "maxpool")}
    sampled = build_model("mean", features, adj)
    for _ in range(a.rounds):
        rnd = {}
        rnd.update(pair("mean_ms", lambda on: ops.csr_aggregate(features, indptr, indices, "mean",
                                                                **({"weights": w} if on else {})), a.iters))
        rnd.update(pair("sum_ms", lambda on: ops.csr_aggregate(grad, t_indptr, t_indices, "sum",
                                                               **({"weights": tw} if on else {})), a.iters))
        rnd.update(pair("max_bwd_ms", lambda on: ops.csr_max_backward(
            z, m_weighted if on else m_plain, dm, indptr, indices, t_indptr, t_indices,
            **({"weights": w, "t_weights": tw} if on else {})), a.iters))
        for kind, m in models.items():
            rnd.update(pair("step_ms_" + kind, lambda on: m.full_neighbor_train_step(
                indptr, indices, train, labels, edge_weight=w if on else None), a.iters))
        rnd.update(pair("sampled_ms_mean", lambda on: sampled.sampled_minibatch_train_step(
            indptr, indices, seeds, seed_labels, edge_weight=w if on else None), a.iters))
        for k in ("plain", "weighted"):
            rnd["mean_GBps_" + k] = res["mean_bytes_" + k] / (rnd["mean_ms_" + k] * 1e-3) / 1e9
        print(json.dumps(rnd), flush=True)
        res["rounds"].append(rnd)
    print(json.dumps({k: v for k, v in res.items() if k != "rounds"}))
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as fp:
        json.dump(res, fp, indent=1)


if __name__ == "__main__":
    main()
