"""The LSTM sequence aggregator's training step (graphsage_seq) at configs[1]'s shape: reddit-shape synthetic graph,
batch 512, 2-hop 25x10, 602 features, dims 128, 41 classes, softmax loss, hidden 128 (model_size="small").

Every round times --steps calls of each of, in this order and on the same batches, between CUDA events: the seq step eager,
the seq step graphed, the graphsage_mean step graphed and the materialised graphsage_maxpool step graphed (the last two for
context).  Then one seq step with torch.cuda.max_memory_allocated reset before it (the peak above what was allocated
before the step), and the three recurrence kernels alone at layer 0 hop 1 (n = 5,120 sequences of k = 25 rows, H = 128)
over --kernel-reps calls between CUDA events, with FLOPs counted from the shapes: the recurrence 2 * n*k * H * 4H per
direction (gs_lstm_forward / gs_lstm_backward), and the bytes of X read by gs_seq_lengths.

    python tools/seq_bench.py --steps 10 --warmup 3 --rounds 2

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
from tools.pool_train_bench import N_CLASSES, _kernel_ms  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--kernel-reps", type=int, default=50)
    ap.add_argument("--math", default=os.environ.get("GS_MATH", "tf32x3"))
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

    def model(kind):
        gs.inits.manual_seed(1)
        sampler = gs.UniformNeighborSampler(adj_dev, seed=123)
        infos = [gs.SAGEInfo("node", sampler, FANOUT[0], DIM), gs.SAGEInfo("node", sampler, FANOUT[1], DIM)]
        return gs.SupervisedGraphsage(N_CLASSES, {"batch_size": BATCH, "dropout": 0.}, table[:, :F], adj_dev, None, infos,
                                      concat=True, aggregator_type=kind, model_size="small", sigmoid_loss=False,
                                      learning_rate=0.01, device=dev)

    peak_model = model("seq")
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    first_loss = float(peak_model.train_step(*inputs[0]))
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    del peak_model
    torch.cuda.empty_cache()

    paths = {"seq_eager": model("seq").train_step, "seq_graphed": model("seq").graphed_train_step(BATCH),
             "mean_graphed": model("mean").graphed_train_step(BATCH),
             "maxpool_graphed": model("maxpool").graphed_train_step(BATCH)}
    for x in inputs[:args.warmup]:
        for fn in paths.values():
            fn(*x)
    torch.cuda.synchronize()
    rounds = [{key: _time(fn, inputs[args.warmup:]) for key, fn in paths.items()} for _ in range(args.rounds)]
    del paths
    torch.cuda.empty_cache()

    # the recurrence kernels alone at layer 0 hop 1
    n, k, H = BATCH * FANOUT[1], FANOUT[0], 128
    X = ops.gather_rows(table[:, :F], torch.from_numpy(rs.randint(0, N_NODES, size=n * k).astype(np.int32)).to(dev))
    kernel = (torch.rand((F + H, 4 * H), device=dev) * 2 - 1) * float(np.sqrt(6.0 / (F + 5 * H)))
    lengths = ops.seq_lengths(X, n, k)
    P = ops.sage_gemm([(X, F, kernel[:F])], math=ops.MATH_TF32X3)
    _, gates, c, _ = ops.lstm_forward(P, kernel[F:], lengths, n, k, train=True)
    dh = torch.randn((n, H), device=dev)
    times = {"seq_lengths": _kernel_ms(lambda: ops.seq_lengths(X, n, k), args.kernel_reps),
             "lstm_forward": _kernel_ms(lambda: ops.lstm_forward(P, kernel[F:], lengths, n, k), args.kernel_reps),
             "lstm_forward_train": _kernel_ms(lambda: ops.lstm_forward(P, kernel[F:], lengths, n, k, train=True),
                                              args.kernel_reps),
             "lstm_backward": _kernel_ms(lambda: ops.lstm_backward(dh, gates, c, lengths, kernel[F:], n, k), args.kernel_reps)}
    rec = 2.0 * n * k * H * 4 * H
    kernels = {key: {"ms": ms} for key, ms in times.items()}
    for key in ("lstm_forward", "lstm_forward_train", "lstm_backward"):
        kernels[key]["tflops"] = rec / (times[key] * 1e-3) / 1e12
    kernels["seq_lengths"]["gb_per_s"] = n * k * F * 4 / (times["seq_lengths"] * 1e-3) / 1e9
    kernels["mean_length"] = float(lengths.float().mean())

    print(json.dumps({"metric": "seq_training_step_ms", "card": _card(), "math": args.math, "steps": args.steps,
                      "warmup": args.warmup, "batch": BATCH, "fanout": FANOUT, "features": F, "dim": DIM, "hidden": H,
                      "rounds": rounds, "seq_peak_bytes_per_step": peak, "seq_first_loss": first_loss,
                      "kernels_layer0_hop1": kernels, "higher_is_better": False,
                      "note": "per round, on the same batches: seq eager, seq graphed, mean graphed, materialised maxpool "
                              "graphed; kernel times include each wrapper's output allocation"}))


if __name__ == "__main__":
    main()
