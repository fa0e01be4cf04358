"""The supervised trainer's step rate against graphed_train_step alone, at configs[1]'s step shape: Reddit-shape synthetic
graph (232,965 nodes, 602 features, 41 classes, 80 / 10 / 10 train / val / test nodes), graphsage_mean, batch 512,
2-hop 25x10, dims 128, softmax loss.

    python tools/train_cli_bench.py

  trainer   supervised_train.train(train_data, flags) for one epoch, fed in memory, with print_every and validate_iter
            larger than the epoch (so only its first step prints and validates); steps / wall second from the loop's
            start to a device synchronise after its last step.
  graphed   model.graphed_train_step(512) replayed on the same epoch's full batches (ids and labels already on the
            device), between CUDA events.

The gap between the two is the host side of the trainer: the iterator's batches and label matrices, the pinned copies
and the launches.  The synthetic graph has a mean degree of about 20 (Reddit's is about 100) so that building the
networkx-style graph and the iterator's tables on the host stays short; the step's shape does not depend on it (the
padded table has max_degree 128 columns either way).  Prints one JSON line with the card's name and power limit read in
the same run.  Single GPU."""
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

N, F, C = 232965, 602, 41


def _card():
    """The card's name and power limit, read now (part of every number this prints)."""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else torch.cuda.get_device_name()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name()


def train_data():
    """load_data's tuple for the synthetic graph: (G, feats [N, F], id_map, walks, class_map)."""
    from graphsage_b200.graph import Graph
    from graphsage_b200.synthetic import community_graph_csr
    indptr, indices, comm = community_graph_csr(N, mean_deg=10, seed=123)
    rs = np.random.RandomState(7)
    kind = rs.choice(3, size=N, p=[0.8, 0.1, 0.1])                # 0 train, 1 val, 2 test
    G = Graph()
    for u in range(N):
        G.add_node(u, val=bool(kind[u] == 1), test=bool(kind[u] == 2))
    for u in range(N):
        for v in indices[indptr[u]:indptr[u + 1]]:
            v = int(v)
            if u < v:
                G.add_edge(u, v, train_removed=bool(kind[u] or kind[v]))
    feats = rs.standard_normal((N, F)).astype(np.float32)
    return G, feats, {u: u for u in range(N)}, [], {u: int(comm[u]) for u in range(N)}


def main():
    assert torch.cuda.is_available(), "needs a CUDA device (no CPU fallback)"
    from graphsage_b200 import supervised_train as sup, train_cli
    dev = torch.device("cuda", 0)
    t0 = time.time()
    data = train_data()
    setup_s = time.time() - t0
    flags = sup.parse_flags(["--model", "graphsage_mean", "--epochs", "1", "--print_every", str(10 ** 9),
                             "--validate_iter", str(10 ** 9), "--gpu", "0", "--base_log_dir", tempfile.mkdtemp(),
                             "--train_prefix", "synthetic/reddit"])
    loop = {}

    def timed_loop(minibatch, flags, step, validate, after):
        torch.cuda.synchronize(dev)
        t = time.time()
        total, costs = train_cli.train_loop(minibatch, flags, step, validate, after)
        torch.cuda.synchronize(dev)
        loop["s"], loop["steps"] = time.time() - t, total
        return total, costs

    sup.train_loop = timed_loop
    model = sup.train(data, flags, device=dev)
    trainer_rate = loop["steps"] / loop["s"]
    del model
    torch.cuda.empty_cache()

    # the same epoch's batches, replayed on a fresh model's graphed step
    minibatch = sup.build_iterator(data, flags)
    feats = np.vstack([data[1], np.zeros((1, F), np.float32)])
    model = sup.build_model(flags, feats, minibatch, minibatch.num_classes, dev)
    minibatch.shuffle()
    batches = []
    while not minibatch.end():
        feed, labels = minibatch.next_minibatch_feed_dict()
        if feed["batch_size"] == flags.batch_size:
            batches.append((torch.tensor(feed["batch"], dtype=torch.int32, device=dev),
                            torch.tensor(labels, dtype=torch.float32, device=dev)))
    step = model.graphed_train_step(flags.batch_size)
    for b in batches[:5]:
        step(*b)
    torch.cuda.synchronize(dev)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for b in batches:
        step(*b)
    e1.record()
    torch.cuda.synchronize(dev)
    graphed_rate = len(batches) / (e0.elapsed_time(e1) / 1e3)
    print(json.dumps({"metric": "supervised_train_steps_per_s", "card": _card(), "config": "configs[1] shape",
                      "nodes": N, "features": F, "classes": C, "batch": flags.batch_size, "fanout": [25, 10],
                      "dims": [128, 128], "trainer_steps": loop["steps"], "trainer_steps_per_s": round(trainer_rate, 1),
                      "graphed_steps": len(batches), "graphed_steps_per_s": round(graphed_rate, 1),
                      "trainer_ms_per_step": round(1e3 / trainer_rate, 3), "graphed_ms_per_step": round(1e3 / graphed_rate, 3),
                      "host_setup_s": round(setup_s, 1), "higher_is_better": True}))


if __name__ == "__main__":
    main()
