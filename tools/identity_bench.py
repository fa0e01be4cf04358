"""The supervised training step with a trainable [N+1, D] node-embedding table (identity_dim = D) at the bench shape
(reddit-shape synthetic graph, graphsage_mean, 2-hop 25x10, batch 512), next to the same step without the table.

    python tools/identity_bench.py --identity-dim 64 [--featureless] --steps 20 --warmup 5

Prints one JSON line (bench_extra.run_train): ms/step with and without the table, the embedding-gradient kernel on its own
(CUDA events, algorithmic bytes) and the dense Adam update of the table.  Single GPU."""
import argparse
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import bench  # noqa: E402
import bench_extra  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--identity-dim", type=int, default=64, help="D: columns of the trainable embedding table (>= 1)")
    ap.add_argument("--featureless", action="store_true", help="the embedding table replaces the features")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--math", default=os.environ.get("GS_MATH", "tf32x3"))
    args = ap.parse_args()
    if args.identity_dim < 1 or args.steps < 1:
        ap.error("--identity-dim and --steps must be >= 1")
    assert torch.cuda.is_available(), "needs a CUDA device (no CPU fallback)"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    bench_extra.run_train(args, bench.build_graph(), 0, 1, 0, None, dev)


if __name__ == "__main__":
    main()
