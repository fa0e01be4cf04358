"""The two-layer max-pool aggregator's neighbour branch at configs[2]'s shape: reddit-shape synthetic graph, bf16 feature
table (F = 602), batch 512, 2-hop 25 x 10, model_size "small" (h1 = 512, h2 = 256).

Timed in one process, alternating over --rounds rounds, between CUDA events over --reps calls after a warm-up:
    k5        K5 (ops.maxpool2_mlp_fused) on layer 0's hop 2: 5,120 groups of k = 25 gathered rows (128,000 rows)
    chain     the unfused bf16 chain on the same rows: gs_gather_rows_f32 -> Dense (bf16 GEMM, bias + ReLU) -> Dense ->
              gs_segment_max, the fp32 [128000, 602], [128000, 512] and [128000, 256] intermediates through HBM
    k4        K4 (ops.maxpool_mlp_fused) of a one-layer max-pool (602 -> 512) on the same rows, for context
    forward   SampleAndAggregate.forward of a graphsage_maxpool-shaped model (dims 128, concat) with aggregator_type
              "twomaxpool" in bf16: both layers, every hop, sampling included
bf16 TFLOP/s = 2 * rows * (F * h1 + h1 * h2) / kernel time (k4: 2 * rows * F * h1).  K5 against the chain: the largest
|difference| over the largest |output| is printed too (they differ in accumulation order only).

    python tools/twomax_bench.py --reps 50 --rounds 3

Prints one JSON line with the card's name and power limit, read in the same run.  Single GPU."""
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


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def _ms(fn, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    if args.reps < 50 or args.rounds < 1 or args.warmup < 1:
        ap.error("--reps >= 50, --rounds >= 1, --warmup >= 1")
    assert torch.cuda.is_available(), "needs a CUDA device (no CPU fallback)"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    import graphsage_b200 as gs
    from graphsage_b200 import ops
    rs = np.random.RandomState(4100)
    g = bench.build_graph()
    table32 = torch.zeros((N_NODES + 1, ops.pad_cols(F)), dtype=torch.float32, device=dev)
    table32[:, :F] = torch.from_numpy(g["features"]).to(dev)
    table = table32.to(torch.bfloat16)[:, :F]
    adj_dev = torch.from_numpy(g["adj"]).to(dev)

    n, k = BATCH * FANOUT[1], FANOUT[0]                  # layer 0, hop 2: 5,120 groups of 25
    rows = n * k
    ids = torch.from_numpy(rs.randint(0, N_NODES, size=rows).astype(np.int32)).to(dev)
    gs.inits.manual_seed(3)
    agg = gs.TwoMaxLayerPoolingAggregator(F, DIM, model_size="small", device="cuda")
    agg.math = ops.MATH_BF16
    for layer in agg.mlp_layers:
        layer.vars["bias"].normal_(0.0, 0.1)
    (W1, b1), (W2, b2) = [(layer.vars["weights"], layer.vars["bias"]) for layer in agg.mlp_layers]
    h1, h2 = W1.shape[1], W2.shape[1]
    p1, p2, pk4 = ops.PackedMlpWeights(), ops.PackedMlpWeights(), ops.PackedMlpWeights()
    out5 = torch.empty((n, h2), device=dev)
    out4 = torch.empty((n, h1), device=dev)
    xbuf = torch.empty((rows, ops.pad_cols(F)), device=dev)[:, :F]

    def k5():
        ops.maxpool2_mlp_fused(table, n, k, W1, b1, p1, W2, b2, p2, row_ids=ids, out=out5)

    def chain():
        x = ops.gather_rows_f32(table, ids=ids, n=rows, out=xbuf)
        return ops.segment_max(agg._mlp(x), n, k)

    def k4():
        ops.maxpool_mlp_fused(table, n, k, W1, b1, pk4, row_ids=ids, out=out4)

    gs.set_default_math("bf16")
    try:
        sampler = gs.UniformNeighborSampler(adj_dev, seed=123)
        infos = [gs.SAGEInfo("node", sampler, FANOUT[0], DIM), gs.SAGEInfo("node", sampler, FANOUT[1], DIM)]
        model = gs.SampleAndAggregate({"batch_size": BATCH, "dropout": 0.}, table, adj_dev, None, infos, concat=True,
                                      aggregator_type="twomaxpool")
    finally:
        gs.set_default_math("fp32")
    seeds = torch.from_numpy(rs.randint(0, N_NODES, size=BATCH).astype(np.int32)).to(dev)

    def forward():
        model.forward(seeds)

    work = {"k5": k5, "chain": chain, "k4": k4, "forward": forward}
    for fn in work.values():
        for _ in range(args.warmup):
            fn()
    torch.cuda.synchronize()
    k5()
    ref = chain()
    torch.cuda.synchronize()
    diff = float((out5 - ref).abs().max() / ref.abs().max())
    times = {name: [] for name in work}
    for _ in range(args.rounds):
        for name, fn in work.items():
            times[name].append(_ms(fn, args.reps))
    flops = {"k5": 2.0 * rows * (F * h1 + h1 * h2), "chain": 2.0 * rows * (F * h1 + h1 * h2), "k4": 2.0 * rows * F * h1}
    res = {"card": _card(), "shape": "configs[2] layer 0 hop 2: %d groups x k=%d, F=%d, h1=%d, h2=%d, bf16 table"
           % (n, k, F, h1, h2), "reps": args.reps, "rounds": args.rounds,
           "k5_vs_chain_max_rel_diff": diff, "peak_mem_mb": torch.cuda.max_memory_allocated() / 2 ** 20}
    for name, ts in times.items():
        best = min(ts)
        res[name + "_ms"] = [round(t, 4) for t in ts]
        if name in flops:
            res[name + "_tflops"] = round(flops[name] / (best * 1e-3) / 1e12, 1)
    res["k5_speedup_vs_chain"] = round(min(times["chain"]) / min(times["k5"]), 2)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
