"""The pooling aggregators' training step, materialised (default) against fused_pool=True, at configs[1]'s shape:
reddit-shape synthetic graph, batch 512, 2-hop 25x10, 602 features, dims 128, 41 classes, softmax loss; hidden 512
(model_size="small") and 1024 ("big").

Per workload (maxpool / meanpool x small / big) four models are built alike: materialised eager, materialised graphed,
fused eager, fused graphed.  Every round times --steps calls of each, in that order, on the same batches, between CUDA
events.  Then, per model size: one step of each path with torch.cuda.max_memory_allocated reset before it (the peak
above what was allocated before the step), and the three backward kernels alone at hop 2 of layer 0 (n = 5,120 groups of
k = 25 gathered rows, K = 602) between CUDA events, with FLOPs counted from the shapes:
    B1 recompute + dpre   2 * n*k * K * hidden     (ops.pool_mlp_backward_dp)
    B2 dWm = X^T dP       2 * n*k * K * hidden     (ops.pool_mlp_backward_dw, with its fixed-order combine)
    B3 dX = dP Wm^T       2 * n*k * 256 * hidden   (ops.pool_mlp_backward_dx; timed at layer 1's input width 256)

    python tools/pool_train_bench.py --steps 10 --warmup 3 --rounds 2

Prints one JSON line, with the card's name and power limit read in the same run.  Single GPU."""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import bench  # noqa: E402
from bench import BATCH, DIM, F, FANOUT, N_NODES  # noqa: E402
from tools.graphed_train_bench import _card, _time  # noqa: E402

N_CLASSES = 41


def _kernel_ms(fn, reps):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--kernel-reps", type=int, default=20)
    ap.add_argument("--math", default=os.environ.get("GS_MATH", "tf32x3"))
    ap.add_argument("--only", default="maxpool/small,meanpool/small,maxpool/big,meanpool/big")
    args = ap.parse_args()
    if args.steps < 1 or args.rounds < 1 or args.warmup < 0 or args.kernel_reps < 1:
        ap.error("--steps, --rounds and --kernel-reps must be >= 1, --warmup >= 0")
    assert torch.cuda.is_available(), "needs a CUDA device (no CPU fallback)"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    import graphsage_b200 as gs
    from graphsage_b200 import ops
    gs.set_default_math(args.math)
    rs = np.random.RandomState(4000)
    g = bench.build_graph()
    table = torch.zeros((N_NODES + 1, ops.pad_cols(F)), dtype=torch.float32, device=dev)
    table[:, :F] = torch.from_numpy(g["features"]).to(dev)
    adj_dev = torch.from_numpy(g["adj"]).to(dev)
    n_in = args.warmup + args.steps
    seeds = rs.randint(0, N_NODES, size=(n_in, BATCH)).astype(np.int64)
    labels = torch.nn.functional.one_hot(torch.from_numpy(g["comm"][seeds.reshape(-1)].astype(np.int64)),
                                         N_CLASSES).float().reshape(n_in, BATCH, N_CLASSES).to(dev)
    ids = torch.from_numpy(seeds.astype(np.int32)).to(dev)
    inputs = [(ids[i], labels[i]) for i in range(n_in)]

    def model(kind, size, fused):
        gs.inits.manual_seed(1)
        sampler = gs.UniformNeighborSampler(adj_dev, seed=123)
        infos = [gs.SAGEInfo("node", sampler, FANOUT[0], DIM), gs.SAGEInfo("node", sampler, FANOUT[1], DIM)]
        return gs.SupervisedGraphsage(N_CLASSES, {"batch_size": BATCH, "dropout": 0.}, table[:, :F], adj_dev, None, infos,
                                      concat=True, aggregator_type=kind, model_size=size, sigmoid_loss=False,
                                      learning_rate=0.01, device=dev, fused_pool=fused)

    results = {}
    for w in args.only.split(","):
        kind, size = w.split("/")
        paths = {}
        for fused in (False, True):
            name = "fused" if fused else "materialised"
            eager, graphed = model(kind, size, fused), model(kind, size, fused)
            paths[name + "_eager"] = eager.train_step
            paths[name + "_graphed"] = graphed.graphed_train_step(BATCH)
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            base = torch.cuda.memory_allocated()
            loss = float(eager.train_step(*inputs[0]))
            torch.cuda.synchronize()
            paths[name + "_peak_bytes"] = torch.cuda.max_memory_allocated() - base
            paths[name + "_first_loss"] = loss
        for x in inputs[:args.warmup]:
            for key in ("materialised_eager", "materialised_graphed", "fused_eager", "fused_graphed"):
                paths[key](*x)
        torch.cuda.synchronize()
        rounds = []
        for _ in range(args.rounds):
            rounds.append({key: _time(paths[key], inputs[args.warmup:])
                           for key in ("materialised_eager", "materialised_graphed", "fused_eager", "fused_graphed")})
        results[w] = {"rounds": rounds,
                      "peak_bytes_per_step": {"materialised": paths["materialised_peak_bytes"],
                                              "fused": paths["fused_peak_bytes"]},
                      "first_step_loss": {"materialised": paths["materialised_first_loss"],
                                          "fused": paths["fused_first_loss"]}}
        del paths
        torch.cuda.empty_cache()

    # the backward kernels alone at hop 2 of layer 0
    kernels = {}
    n, k, K = BATCH * FANOUT[1], FANOUT[0], F
    tb = ops.cast_rows_bf16(table[:, :F])
    row_ids = torch.from_numpy(rs.randint(0, N_NODES, size=n * k).astype(np.int32)).to(dev)
    for size, hidden in (("small", 512), ("big", 1024)):
        W = torch.randn((K, hidden), device=dev) * 0.05
        b = torch.randn((hidden,), device=dev) * 0.1
        dhp = torch.randn((n, hidden), device=dev)
        packed = ops.PackedMlpWeights()
        grad = ops.pool_mlp_backward_dp(tb, n, k, W, b, packed, dhp, row_ids=row_ids, K=K)
        dW, db = torch.zeros_like(W), torch.zeros_like(b)
        W1 = torch.randn((256, hidden), device=dev) * 0.05
        pdx = ops.PackedMlpDxWeights(256)
        times = {
            "B1": _kernel_ms(lambda: ops.pool_mlp_backward_dp(tb, n, k, W, b, packed, dhp, row_ids=row_ids, K=K),
                             args.kernel_reps),
            "B2": _kernel_ms(lambda: ops.pool_mlp_backward_dw(tb, n, k, grad, dW, db, row_ids=row_ids, K=K), args.kernel_reps),
            "B3": _kernel_ms(lambda: ops.pool_mlp_backward_dx(grad, n, k, W1, pdx), args.kernel_reps),
        }
        flops = {"B1": 2.0 * n * k * K * hidden, "B2": 2.0 * n * k * K * hidden, "B3": 2.0 * n * k * 256 * hidden}
        kernels[size] = {key: {"ms": times[key], "tflops": flops[key] / (times[key] * 1e-3) / 1e12} for key in times}

    print(json.dumps({"metric": "pool_training_step_ms", "card": _card(), "math": args.math, "steps": args.steps,
                      "warmup": args.warmup, "batch": BATCH, "fanout": FANOUT, "features": F, "dim": DIM,
                      "results": results, "kernels_hop2_layer0": kernels, "higher_is_better": False,
                      "note": "per round, on the same batches: materialised eager, materialised graphed, fused eager, fused "
                              "graphed; kernel times include each wrapper's workspace allocation"}))


if __name__ == "__main__":
    main()
