"""Time the full-batch training step (SupervisedGraphsage.full_neighbor_train_step) and its parts on the GPU, against one
sampled epoch over the same nodes.

    python tools/full_neighbor_train_bench.py [--iters 5] [--rounds 2] [--out full_neighbor_train_bench.json]

Input: community_graph_csr(232,965, mean_deg=50) (Reddit's node count and density) with 602 random fp32 features and 41
classes; the train nodes are a fixed random 66 % of the nodes.  Model: 2 layers, concat, width 128 per half, tf32x3
combine GEMMs, mean and max-pool.  Per aggregator, after one warm-up step (which builds and caches the transposes):
  transpose_ms   one ops.csr_transpose build (CUDA events), without and with self entries;
  forward_ms     full_neighbor_loss (CUDA events around it);
  backward_ms    loss.backward(); of it, reductions_ms is the sum of the probed CSR kernels (csr_aggregate "sum",
                 csr_max_backward, the last layer's embedding_grad scatter) and gemm_other_ms the rest (the weight and
                 source GEMMs, ReLU masks, divisions);
  adam_ms        clipping and optimizer.step();
  step_ms        full_neighbor_train_step end to end (events, --iters steps);
  peak_MB        torch.cuda.max_memory_allocated during one step, above the resident set;
  sampled_epoch_s  train_step over every train node in batches of 512 (fanouts 25, 10), with a device synchronise.
Everything is measured --rounds times in one process; the card name and power limit are read in the same command."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import graphsage_b200 as gs  # noqa: E402
from graphsage_b200 import ops  # noqa: E402
from graphsage_b200.minibatch import padded_from_csr_fast  # noqa: E402
from graphsage_b200.synthetic import community_graph_csr  # noqa: E402

F, C = 602, 41
REDUCTIONS = ("csr_aggregate/", "csr_max_backward/", "embedding_grad/")


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


def probed_ms(prefixes):
    torch.cuda.synchronize()
    total = sum(e0.elapsed_time(e1) for name, evs in (ops.PROBE or {}).items() if name.startswith(prefixes)
                for e0, e1 in evs)
    ops.PROBE = None
    return total


def build_model(kind, features, adj):
    gs.set_default_math("tf32x3")
    gs.inits.manual_seed(1)
    sampler = gs.UniformNeighborSampler(adj, seed=123)
    infos = [gs.SAGEInfo("node", sampler, 25, 128), gs.SAGEInfo("node", sampler, 10, 128)]
    m = gs.SupervisedGraphsage(C, {"batch_size": 512, "dropout": 0.}, features, adj, None, infos, concat=True,
                               aggregator_type=kind, learning_rate=0.01)
    gs.set_default_math("fp32")
    return m


def measure(kind, features, adj, indptr, indices, train, labels, iters):
    m = build_model(kind, features, adj)
    res = {"aggregator": kind, "train_nodes": int(train.numel())}
    m.full_neighbor_train_step(indptr, indices, train, labels)                 # warm-up: transposes cached, Adam state
    for with_self in (False, True):
        with Timer() as t:
            ops.csr_transpose(indptr, indices, with_self=with_self)
        res["transpose%s_ms" % ("_self" if with_self else "")] = t.ms
    with Timer() as t:
        loss = m.full_neighbor_loss(indptr, indices, train, labels)
    res["forward_ms"] = t.ms
    m.optimizer.zero_grad(set_to_none=True)
    ops.PROBE = {}
    with Timer() as t:
        loss.backward()
    res["backward_ms"] = t.ms
    res["reductions_ms"] = probed_ms(REDUCTIONS)
    res["gemm_other_ms"] = res["backward_ms"] - res["reductions_ms"]
    with Timer() as t:
        for p in m.parameters():
            if p.grad is not None:
                p.grad.clamp_(-5.0, 5.0)
        m.optimizer.step()
    res["adam_ms"] = t.ms
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    with Timer() as t:
        for _ in range(iters):
            m.full_neighbor_train_step(indptr, indices, train, labels)
    res["step_ms"] = t.ms / iters
    res["peak_MB"] = (torch.cuda.max_memory_allocated() - base) / 2**20
    ids = train.cpu()
    lab = labels
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(0, ids.numel(), 512):
        m.train_step(ids[i:i + 512], lab[i:i + 512])
    torch.cuda.synchronize()
    res["sampled_epoch_s"] = time.perf_counter() - t0
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--out", default="full_neighbor_train_bench.json")
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
    g = torch.Generator(device="cuda").manual_seed(0)
    t = torch.zeros((n + 1, ops.pad_cols(F)), dtype=torch.float32, device="cuda")
    t[:-1, :F] = torch.randn((n, F), generator=g, device="cuda")
    features = t[:, :F]
    adj = torch.from_numpy(padded_from_csr_fast(ip, ix, 128)[0]).cuda()
    indptr, indices = torch.from_numpy(ip).cuda(), torch.from_numpy(ix).cuda()
    for _ in range(a.rounds):
        rnd = [measure(kind, features, adj, indptr, indices, train, labels, a.iters) for kind in ("mean", "maxpool")]
        for r in rnd:
            print(json.dumps(r), flush=True)
        res["rounds"].append(rnd)
    print(json.dumps({k: v for k, v in res.items() if k != "rounds"}))
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as fp:
        json.dump(res, fp, indent=1)


if __name__ == "__main__":
    main()
