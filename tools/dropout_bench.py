"""Cost of training dropout at the bench shape (reddit-shape synthetic graph, graphsage_mean, 2-hop 25x10, batch 512, 41
classes): the supervised training step at placeholders['dropout'] = 0 and = --rate, and the layer-0 fused gather with
masks (gs_gather_mean_dropout) against the plain one (gs_gather_mean) on the segments of a real step.  Each pair is timed
alternately in one process (--rounds rounds of --steps steps each), so clock drift hits both sides alike.

    python tools/dropout_bench.py --rate 0.5 --steps 20 --warmup 5 --rounds 3

Prints one JSON line.  Single GPU."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import bench  # noqa: E402
import bench_extra  # noqa: E402
from bench import BATCH, DIM, F, FANOUT, N_NODES  # noqa: E402


def _card():
    """The card's name and power limit, read now (part of every number this prints)."""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else torch.cuda.get_device_name()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name()


def _time(fn, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rate", type=float, default=0.5)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--math", default=os.environ.get("GS_MATH", "tf32x3"))
    args = ap.parse_args()
    if not 0.0 < args.rate < 1.0 or args.steps < 1 or args.rounds < 1:
        ap.error("--rate must be in (0, 1), --steps and --rounds >= 1")
    assert torch.cuda.is_available(), "needs a CUDA device (no CPU fallback)"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    import graphsage_b200 as gs
    from graphsage_b200 import ops
    gs.set_default_math(args.math)
    g = bench.build_graph()
    table = torch.zeros((N_NODES + 1, ops.pad_cols(F)), dtype=torch.float32, device=dev)
    table[:, :F] = torch.from_numpy(g["features"]).to(dev)
    adj_dev = torch.from_numpy(g["adj"]).to(dev)

    def make_model(rate):
        sampler = gs.UniformNeighborSampler(adj_dev, seed=123)
        infos = [gs.SAGEInfo("node", sampler, FANOUT[0], DIM), gs.SAGEInfo("node", sampler, FANOUT[1], DIM)]
        return gs.SupervisedGraphsage(41, {"batch_size": BATCH, "dropout": rate}, table[:, :F], adj_dev, None, infos, concat=True,
                                      aggregator_type="mean", sigmoid_loss=False, learning_rate=0.01, device=dev)

    models = {0.0: make_model(0.0), args.rate: make_model(args.rate)}
    rs = np.random.RandomState(4000)
    total = args.warmup + args.steps
    seeds = torch.from_numpy(rs.randint(0, N_NODES, size=(total, BATCH)).astype(np.int32)).to(dev)
    labels = torch.nn.functional.one_hot(torch.from_numpy(g["comm"][seeds.cpu().numpy().reshape(-1)].astype(np.int64)),
                                         41).float().reshape(total, BATCH, 41).to(dev)
    step_ms = {0.0: [], args.rate: []}
    for _ in range(args.rounds):
        for rate, m in models.items():
            ms, _, _ = bench_extra._timed_train_steps(m, seeds, labels, args, None, dev)
            step_ms[rate].append(ms / args.steps)

    # the layer-0 segments and sites of one real dropout step, replayed through the two gathers alone
    seen = {}
    real = ops.gather_mean_dropout

    def keep(src, segments, ns, ss, **kw):
        if "segs" not in seen:
            seen.update(src=src, segs=segments, ns=ns, ss=ss)
        return real(src, segments, ns, ss, **kw)

    ops.gather_mean_dropout = keep
    try:
        models[args.rate].train_step(seeds[0], labels[0])
    finally:
        ops.gather_mean_dropout = real
    src, segs, ns, ss = seen["src"], seen["segs"], seen["ns"], seen["ss"]
    rows = sum(s.n for s in segs)
    gathered = sum(s.n * (s.k + 1) for s in segs)
    nbytes = gathered * F * 4 + 2 * rows * ops.pad_cols(F) * 4          # rows read + self and mean rows written
    reps = 50
    plain = lambda: ops.gather_mean(src, segs, want_self=True)          # noqa: E731
    masked = lambda: ops.gather_mean_dropout(src, segs, ns, ss, want_self=True)   # noqa: E731
    for _ in range(5):
        plain()
        masked()
    us = {"plain": [], "masked": []}
    for _ in range(args.rounds):
        us["plain"].append(_time(plain, reps) * 1e3)
        us["masked"].append(_time(masked, reps) * 1e3)
    best = {k: min(v) for k, v in us.items()}
    print(json.dumps({
        "metric": "training_step_ms", "workload": "supervised graphsage_mean training step (fwd + bwd + clipped Adam), "
        "reddit-shape synthetic, 2-hop 25x10, batch %d, 41 classes, dropout 0 vs %g" % (BATCH, args.rate),
        "card": _card(), "rate": args.rate, "steps": args.steps, "warmup": args.warmup, "rounds": args.rounds,
        "ms_per_step_p0": step_ms[0.0], "ms_per_step_dropout": step_ms[args.rate],
        "gather_layer0": {"rows": rows, "gathered_rows": gathered, "columns": F, "algorithmic_bytes": nbytes,
                          "us_plain": us["plain"], "us_masked": us["masked"],
                          "TB_per_s_plain": nbytes / (best["plain"] * 1e-6) / 1e12,
                          "TB_per_s_masked": nbytes / (best["masked"] * 1e-6) / 1e12},
        "higher_is_better": False, "dtype": "f32", "data": "synthetic",
        "note": "the two step timings alternate per round in one process on the same seeds; the gathers replay the layer-0 "
                "segments and sites of one real dropout step, 50 calls per timing, best round used for TB/s"}))


if __name__ == "__main__":
    main()
