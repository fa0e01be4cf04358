"""Time minibatch training over whole neighbourhoods (SupervisedGraphsage.full_neighbor_minibatch_train_step) on the GPU,
against the whole-graph step on the same ids and a sampled step of the same batch size.

    python tools/full_neighbor_minibatch_bench.py [--iters 5] [--rounds 2] [--out full_neighbor_minibatch_bench.json]

Graphs: "reddit", community_graph_csr(232,965, mean_deg=50) (Reddit's node count and density: a 512-node batch's
receptive field is a large, hub-heavy share of it) with 602 random fp32 features, and "sparse",
community_graph_csr(2,000,000, mean_deg=10) with 128 features (the regime where the receptive field is small).  Model: 2
layers, concat, width 128 per half, tf32x3 combine GEMMs, 41 classes; mean and max-pool; batches of 512 and 4096 random
node ids.  Per case, after one warm-up of each step:
  V, entries      |V_0|, |V_1| and the entries of blocks 0 and 1 (|V_2| is the batch);
  blocks_ms       one ops.csr_blocks call, its device-to-host read of the sizes included (CUDA events);
  forward_ms      full_neighbor_minibatch_loss (the blocks included);  backward_ms  loss.backward() (the block
                  transposes included);  step_ms  full_neighbor_minibatch_train_step end to end (--iters steps);
  peak_MB         torch.cuda.max_memory_allocated during one step, above the resident set;
  whole_step_ms / whole_peak_MB   full_neighbor_train_step on the same ids (its transposes cached by the warm-up);
                  "oom" if it does not fit;
  sampled_step_ms train_step on the same ids (fanouts 25, 10).
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

C = 41
GRAPHS = (("reddit", 232965, 50, 602), ("sparse", 2000000, 10, 128))


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
    infos = [gs.SAGEInfo("node", sampler, 25, 128), gs.SAGEInfo("node", sampler, 10, 128)]
    m = gs.SupervisedGraphsage(C, {"batch_size": 512, "dropout": 0.}, features, adj, None, infos, concat=True,
                               aggregator_type=kind, learning_rate=0.01)
    gs.set_default_math("fp32")
    return m


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
    res = {"aggregator": kind, "batch": int(ids.numel())}
    blocks = ops.csr_blocks(indptr, indices, ids, 2)
    res["V"] = [int(b.src_ids.numel()) for b in blocks]
    res["entries"] = [int(b.indices.numel()) for b in blocks]
    del blocks
    with Timer() as t:
        ops.csr_blocks(indptr, indices, ids, 2)
    res["blocks_ms"] = t.ms
    m.full_neighbor_minibatch_train_step(indptr, indices, ids, labels)            # warm-up: Adam state
    with Timer() as t:
        loss = m.full_neighbor_minibatch_loss(indptr, indices, ids, labels)
    res["forward_ms"] = t.ms
    m.optimizer.zero_grad(set_to_none=True)
    with Timer() as t:
        loss.backward()
    res["backward_ms"] = t.ms
    del loss
    res["step_ms"], res["peak_MB"] = timed_steps(
        lambda: m.full_neighbor_minibatch_train_step(indptr, indices, ids, labels), iters)
    try:
        m.full_neighbor_train_step(indptr, indices, ids, labels)                   # warm-up: transposes cached
        res["whole_step_ms"], res["whole_peak_MB"] = timed_steps(
            lambda: m.full_neighbor_train_step(indptr, indices, ids, labels), iters)
    except torch.cuda.OutOfMemoryError:
        res["whole_step_ms"] = res["whole_peak_MB"] = "oom"
    m._full_neighbor_graph = None
    torch.cuda.empty_cache()
    host_ids, host_labels = ids.cpu(), labels
    m.train_step(host_ids, host_labels)
    res["sampled_step_ms"], _ = timed_steps(lambda: m.train_step(host_ids, host_labels), iters)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--out", default="full_neighbor_minibatch_bench.json")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "the benchmark needs a CUDA device"
    gs._lib.lib()
    res = {"card": card(), "graphs": {}, "rounds": [[] for _ in range(a.rounds)]}
    print(json.dumps({"card": res["card"]}), flush=True)
    for name, n_nodes, deg, F in GRAPHS:
        ip, ix, _ = community_graph_csr(n_nodes, mean_deg=deg)
        n = len(ip) - 1
        res["graphs"][name] = {"nodes": n, "entries": int(ip[-1]), "max_degree": int(np.diff(ip).max()), "features": F}
        g = torch.Generator(device="cuda").manual_seed(0)
        t = torch.zeros((n + 1, ops.pad_cols(F)), dtype=torch.float32, device="cuda")
        t[:-1, :F] = torch.randn((n, F), generator=g, device="cuda")
        features = t[:, :F]
        adj = torch.from_numpy(padded_from_csr_fast(ip, ix, 128)[0]).cuda()
        indptr, indices = torch.from_numpy(ip).cuda(), torch.from_numpy(ix).cuda()
        rs = np.random.RandomState(0)
        for r in range(a.rounds):
            for kind in ("mean", "maxpool"):
                for batch in (512, 4096):
                    ids = torch.from_numpy(rs.choice(n, batch, replace=False).astype(np.int32)).cuda()
                    labels = torch.zeros((batch, C), device="cuda")
                    labels[torch.arange(batch, device="cuda"), torch.from_numpy(rs.randint(0, C, batch)).cuda()] = 1.0
                    out = dict(graph=name, round=r, **measure(kind, features, adj, indptr, indices, ids, labels, a.iters))
                    print(json.dumps(out), flush=True)
                    res["rounds"][r].append(out)
        del t, features, adj, indptr, indices
        torch.cuda.empty_cache()
    print(json.dumps({k: v for k, v in res.items() if k != "rounds"}))
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as fp:
        json.dump(res, fp, indent=1)


if __name__ == "__main__":
    main()
