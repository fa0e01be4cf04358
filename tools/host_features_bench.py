"""Training from a feature table in host memory (HostFeatures) against the same table in HBM.

Workload: the Reddit-shape synthetic graph of bench.py (232,965 nodes, 602 fp32 features), SupervisedGraphsage with the
mean aggregator, fanouts 25 x 10, dims 128, batch 512, 41 classes.  For every cache fraction (the hottest rows by
host_features.hot_rows held on the device) it reports:

    ms per training step and seeds/s, host table and device table, timed alternately in the same run (CUDA events);
    staged rows per step (the distinct uncached rows a step fetched, read from the device count after each step);
    fetch-kernel ms (CUDA events around gs_host_fetch, a separate pass with the probes on) and the host-link rate
    staged bytes / fetch time.

    python tools/host_features_bench.py --steps 20 --warmup 3 --rounds 3

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

N_CLASSES = 41


def _card():
    """The card's name, power limit and PCIe link, read now (part of every number this prints)."""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,pcie.link.gen.current,pcie.link.width.current",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
        return out.splitlines()[0] if out else torch.cuda.get_device_name()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name()


def _time(fn, inputs):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for x in inputs:
        fn(*x)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / len(inputs)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--fractions", default="0,0.1,0.25,0.5,1")
    ap.add_argument("--math", default=os.environ.get("GS_MATH", "tf32x3"))
    args = ap.parse_args()
    if args.steps < 1 or args.rounds < 1 or args.warmup < 0:
        ap.error("--steps and --rounds must be >= 1, --warmup >= 0")
    assert torch.cuda.is_available(), "needs a CUDA device (no CPU fallback)"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    import graphsage_b200 as gs
    from graphsage_b200 import ops
    from graphsage_b200.host_features import hot_rows
    gs.set_default_math(args.math)
    card = _card()
    g = bench.build_graph()
    feats = np.zeros((N_NODES + 1, F), np.float32)
    feats[:N_NODES] = g["features"][:N_NODES]
    table = torch.zeros((N_NODES + 1, ops.pad_cols(F)), dtype=torch.float32, device=dev)
    table[:, :F] = torch.from_numpy(feats).to(dev)
    adj_dev = torch.from_numpy(g["adj"]).to(dev)
    rs = np.random.RandomState(4000)
    n_in = args.warmup + args.steps
    seeds = rs.randint(0, N_NODES, size=(n_in, BATCH))
    labels = torch.nn.functional.one_hot(torch.from_numpy(g["comm"][seeds.reshape(-1)].astype(np.int64)), N_CLASSES)
    labels = labels.float().reshape(n_in, BATCH, N_CLASSES).to(dev)
    ids = torch.from_numpy(seeds.astype(np.int32)).to(dev)
    inputs = [(ids[i], labels[i]) for i in range(n_in)]

    def model(features):
        gs.inits.manual_seed(1)
        sampler = gs.UniformNeighborSampler(adj_dev, seed=123)
        infos = [gs.SAGEInfo("node", sampler, FANOUT[0], DIM), gs.SAGEInfo("node", sampler, FANOUT[1], DIM)]
        return gs.SupervisedGraphsage(N_CLASSES, {"batch_size": BATCH, "dropout": 0.}, features, adj_dev, None, infos,
                                      concat=True, aggregator_type="mean", learning_rate=0.01, device=dev)

    rows_per_step = BATCH * (1 + FANOUT[1] + FANOUT[1] * FANOUT[0])
    results = {}
    for frac in [float(x) for x in args.fractions.split(",")]:
        hf = gs.HostFeatures(torch.from_numpy(feats), cache_ids=hot_rows(g["adj"], int(round(frac * N_NODES))))
        host_m, dev_m = model(hf), model(table[:, :F])
        for x in inputs[:args.warmup]:
            host_m.train_step(*x)
            dev_m.train_step(*x)
        torch.cuda.synchronize()
        timed = inputs[args.warmup:]
        rounds = [{"host_ms": _time(host_m.train_step, timed), "device_ms": _time(dev_m.train_step, timed)}
                  for _ in range(args.rounds)]
        # a separate pass with the fetch probe on: kernel time and the rows each step staged
        ops.PROBE, staged = {}, []
        try:
            for x in timed:
                host_m.train_step(*x)
                dev_m.train_step(*x)                 # both models stay on the same step for the comparison below
                staged.append(int(hf.count))
            torch.cuda.synchronize()
            fetch_ms = [e0.elapsed_time(e1) for e0, e1 in ops.PROBE.get("host_fetch", [])]
        finally:
            ops.PROBE = None
        same = bool(torch.equal(host_m.train_step(*timed[0]), dev_m.train_step(*timed[0])))
        # control: a second device-table model through the same steps - are two device-table runs bit-identical here?
        twin = model(table[:, :F])
        for x in inputs[:args.warmup] + timed * (args.rounds + 1) + timed[:1]:
            twin.train_step(*x)
        same_twin = bool(torch.equal(twin.train_step(*timed[0]), dev_m.train_step(*timed[0])))
        del twin
        host_ms = float(np.median([r["host_ms"] for r in rounds]))
        dev_ms = float(np.median([r["device_ms"] for r in rounds]))
        f_ms = float(np.median(fetch_ms))
        rows = float(np.mean(staged))
        results[str(frac)] = {
            "cached_rows": hf.n_cached, "rounds": rounds,
            "host_ms": host_ms, "device_ms": dev_ms,
            "host_seeds_per_s": BATCH / host_ms * 1e3, "device_seeds_per_s": BATCH / dev_ms * 1e3,
            "staged_rows_per_step": rows, "sampled_rows_per_step": rows_per_step,
            "fetch_ms": f_ms, "host_link_GBps": rows * hf.row_bytes / (f_ms * 1e-3) / 1e9,
            "same_loss_as_device_table": same, "device_table_twice_same_loss": same_twin}
        hf.close()
        del host_m, dev_m, hf
        torch.cuda.empty_cache()

    print(json.dumps({"metric": "host_table_training_step_ms", "card": card, "math": args.math, "steps": args.steps,
                      "warmup": args.warmup, "batch": BATCH, "fanout": FANOUT, "dim": DIM, "features": F,
                      "row_bytes": ops.pad_cols(F) * 4, "results": results, "higher_is_better": False}))


if __name__ == "__main__":
    main()
