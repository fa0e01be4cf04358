"""Eager train_step against its CUDA-graph replay (model.graphed_train_step) at user-sized shapes:

    sup_mean      SupervisedGraphsage, graphsage_mean - configs[1]: reddit-shape synthetic graph, batch 512, 2-hop 25x10,
                  dims 128, 41 classes, softmax loss
    sup_maxpool   the same with the max-pool aggregator
    unsup_mean    UnsupervisedGraphsage, graphsage_mean, same graph, batch 512, 20 negatives
    n2v           Node2VecModel at the shape of tools/n2v_bench.py (V = 232,966, d = 256, batch 512, 20 negatives)

Each workload builds two models alike: one trained by the eager train_step (the default, non-capturable Adam) and one by
the replayed step.  Every round times --steps eager steps, then --steps replays, between CUDA events, on the same
batches, so drift hits both sides alike.

    python tools/graphed_train_bench.py --steps 30 --warmup 5 --rounds 3

Prints one JSON line, with the card's name and power limit read in the same run.  Single GPU."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import bench  # noqa: E402
from bench import BATCH, DIM, F, FANOUT, N_NODES  # noqa: E402

N_CLASSES, NEG = 41, 20
N2V_V, N2V_D = 232966, 256


def _card():
    """The card's name and power limit, read now (part of every number this prints)."""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else torch.cuda.get_device_name()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name()


def _time(fn, inputs):
    """Milliseconds per step of fn(*inputs[i]) over every i, between two CUDA events."""
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for x in inputs:
        fn(*x)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / len(inputs)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--math", default=os.environ.get("GS_MATH", "tf32x3"))
    ap.add_argument("--only", default="sup_mean,sup_maxpool,unsup_mean,n2v")
    ap.add_argument("--table", choices=["fp32", "bf16", "int8"], default="fp32",
                    help="the feature table the graphsage models read: fp32, bf16, or int8 rows with a per-row scale")
    args = ap.parse_args()
    if args.steps < 1 or args.rounds < 1 or args.warmup < 0:
        ap.error("--steps and --rounds must be >= 1, --warmup >= 0")
    assert torch.cuda.is_available(), "needs a CUDA device (no CPU fallback)"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    import graphsage_b200 as gs
    from graphsage_b200 import ops
    gs.set_default_math(args.math)
    only = args.only.split(",")
    rs = np.random.RandomState(4000)
    n_in = args.warmup + args.steps
    results = {}

    g = None
    if any(w != "n2v" for w in only):
        g = bench.build_graph()
        table = torch.zeros((N_NODES + 1, ops.pad_cols(F)), dtype=torch.float32, device=dev)
        table[:, :F] = torch.from_numpy(g["features"]).to(dev)
        adj_dev = torch.from_numpy(g["adj"]).to(dev)
        features = {"fp32": lambda: table[:, :F], "bf16": lambda: table.to(torch.bfloat16)[:, :F],
                    "int8": lambda: gs.Int8Features(table[:, :F])}[args.table]()

    def sage(kind, supervised):
        gs.inits.manual_seed(1)
        sampler = gs.UniformNeighborSampler(adj_dev, seed=123)
        infos = [gs.SAGEInfo("node", sampler, FANOUT[0], DIM), gs.SAGEInfo("node", sampler, FANOUT[1], DIM)]
        if supervised:
            return gs.SupervisedGraphsage(N_CLASSES, {"batch_size": BATCH, "dropout": 0.}, features, adj_dev, None, infos,
                                          concat=True, aggregator_type=kind, sigmoid_loss=False, learning_rate=0.01, device=dev)
        return gs.UnsupervisedGraphsage({"batch_size": BATCH, "dropout": 0.}, features, adj_dev, g["deg"][:N_NODES], infos,
                                        concat=True, aggregator_type=kind, neg_sample_size=NEG, learning_rate=1e-5, device=dev)

    def sage_inputs(supervised):
        seeds = rs.randint(0, N_NODES, size=(n_in, BATCH)).astype(np.int64)
        a = torch.from_numpy(seeds.astype(np.int32)).to(dev)
        if supervised:
            b = torch.nn.functional.one_hot(torch.from_numpy(g["comm"][seeds.reshape(-1)].astype(np.int64)),
                                            N_CLASSES).float().reshape(n_in, BATCH, N_CLASSES).to(dev)
        else:
            b = torch.from_numpy(rs.randint(0, N_NODES, size=(n_in, BATCH)).astype(np.int32)).to(dev)
        return [(a[i], b[i]) for i in range(n_in)]

    def n2v_pair():
        r = np.random.RandomState(0)
        deg = np.minimum(r.pareto(1.5, size=N2V_V - 1) * 5 + 1, 20000).astype(np.int64).astype(np.float64)
        pool = r.randint(0, N2V_V - 1, size=BATCH * 16)
        inputs = [(torch.from_numpy(r.choice(pool, BATCH).astype(np.int32)).to(dev),
                   torch.from_numpy(r.choice(pool, BATCH).astype(np.int32)).to(dev)) for _ in range(n_in)]
        make = lambda: gs.Node2VecModel({"batch_size": BATCH}, N2V_V, deg, nodevec_dim=N2V_D, lr=0.01,  # noqa: E731
                                        neg_sample_size=NEG, seed=1, device=dev)
        return make(), make(), inputs

    for w in only:
        if w == "n2v":
            eager, graphed, inputs = n2v_pair()
        else:
            kind = "maxpool" if w == "sup_maxpool" else "mean"
            sup = w.startswith("sup")
            eager, graphed, inputs = sage(kind, sup), sage(kind, sup), sage_inputs(sup)
        step = graphed.graphed_train_step(BATCH)
        for x in inputs[:args.warmup]:
            eager.train_step(*x)
            step(*x)
        torch.cuda.synchronize()
        timed = inputs[args.warmup:]
        rounds = []
        for _ in range(args.rounds):
            rounds.append({"eager_ms": _time(eager.train_step, timed), "graphed_ms": _time(step, timed)})
        loss_e, loss_g = float(eager.train_step(*timed[0])), float(step(*timed[0]).clone())
        results[w] = {"rounds": rounds, "finite": bool(np.isfinite(loss_e) and np.isfinite(loss_g))}
        del eager, graphed, step
        torch.cuda.empty_cache()

    print(json.dumps({"metric": "training_step_ms", "card": _card(), "math": args.math, "table": args.table, "steps": args.steps,
                      "warmup": args.warmup, "batch": BATCH, "fanout": FANOUT, "dim": DIM, "results": results,
                      "higher_is_better": False,
                      "note": "per round: --steps eager train_step calls, then --steps replays of graphed_train_step, on the "
                              "same batches; separate models built alike (eager: default Adam; graphed: capturable Adam)"}))


if __name__ == "__main__":
    main()
