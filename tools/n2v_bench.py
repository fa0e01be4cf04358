"""Cost of the Node2Vec / DeepWalk training step at the Reddit shape (V = 232,966 table rows, nodevec_dim = 256, batch 512,
20 unique negatives): Node2VecModel.train_step (gs_sample_unigram_unique + gs_skipgram_grad + 2 x gs_embedding_sgd)
against an eager torch-GPU restatement of the same step (lookups, autograd, index_add_ SGD), timed alternately in one
process (--rounds rounds of --steps steps each), then every new kernel on its own with CUDA events (--reps calls each).
The pairs are seeded and repeat ids (a walk corpus does); the degrees are a seeded power law.

    python tools/n2v_bench.py --steps 50 --warmup 10 --rounds 3

Prints one JSON line, with the card's name and power limit read in the same run.  Single GPU."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from graphsage_b200 import ops  # noqa: E402
from graphsage_b200.node2vec import Node2VecModel  # noqa: E402

V, D, B, S = 232966, 256, 512, 20


def _card():
    """The card's name and power limit, read now (part of every number this prints)."""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else torch.cuda.get_device_name()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name()


def _time(fn, reps):
    """Mean milliseconds per call of `reps` back-to-back calls between two CUDA events."""
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


class TorchStep(object):
    """The same step in eager torch: embedding lookups, the biased loss, autograd, sparse SGD through index_add_."""

    def __init__(self, model):
        self.T = model.target_embeds.clone()
        self.C = model.context_embeds.clone()
        self.b = model.context_bias.clone()
        self.lr = model.lr
        self.sampler = model.neg_sampler

    def __call__(self, b1, b2):
        neg = self.sampler().long()
        b1, b2 = b1.long(), b2.long()
        t = self.T[b1].requires_grad_()
        c = self.C[b2].requires_grad_()
        n = self.C[neg].requires_grad_()
        cb, nb = self.b[b2].requires_grad_(), self.b[neg].requires_grad_()
        aff = (t * c).sum(1) + cb
        neg_aff = t @ n.t() + nb[None, :]
        loss = (torch.nn.functional.softplus(-aff).sum() + torch.nn.functional.softplus(neg_aff).sum()) / b1.numel()
        loss.backward()
        with torch.no_grad():
            self.T.index_add_(0, b1, t.grad, alpha=-self.lr)
            self.C.index_add_(0, b2, c.grad, alpha=-self.lr)
            self.C.index_add_(0, neg, n.grad, alpha=-self.lr)
            self.b.index_add_(0, b2, cb.grad, alpha=-self.lr)
            self.b.index_add_(0, neg, nb.grad, alpha=-self.lr)
        return loss.detach()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=200)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    r = np.random.RandomState(0)
    deg = np.minimum(r.pareto(1.5, size=V - 1) * 5 + 1, 20000).astype(np.int64).astype(np.float64)   # N degrees, N + 1 rows
    n_batches = 64
    pool = r.randint(0, V - 1, size=B * n_batches // 4)                   # a quarter as many distinct ids as pair slots
    pairs = [(torch.from_numpy(r.choice(pool, B).astype(np.int32)).cuda(),
              torch.from_numpy(r.choice(pool, B).astype(np.int32)).cuda()) for _ in range(n_batches)]
    model = Node2VecModel({"batch_size": B}, V, deg, nodevec_dim=D, lr=0.01, neg_sample_size=S, seed=1)
    ref = TorchStep(model)
    k = {"i": 0}

    def ours():
        b1, b2 = pairs[k["i"] % n_batches]
        k["i"] += 1
        return model.train_step(b1, b2)

    def theirs():
        b1, b2 = pairs[k["i"] % n_batches]
        k["i"] += 1
        return ref(b1, b2)

    for _ in range(args.warmup):
        ours()
        theirs()
    torch.cuda.synchronize()
    rounds = []
    for _ in range(args.rounds):
        rounds.append({"train_step_ms": _time(ours, args.steps), "torch_eager_ms": _time(theirs, args.steps)})

    # the kernels on their own, on one batch of the same shape
    b1, b2 = pairs[0]
    neg = model.neg_sampler()
    ctx = model._context[:, :D + 1]
    out = ops.skipgram_grad(model.target_embeds, ctx, b1, b2, neg)
    kernels = {
        "sample_unigram_unique_us": 1e3 * _time(lambda: ops.sample_unigram_unique(model.neg_sampler.cdf, S, 1, 0), args.reps),
        "skipgram_grad_us": 1e3 * _time(lambda: ops.skipgram_grad(model.target_embeds, ctx, b1, b2, neg), args.reps),
        "embedding_sgd_target_us": 1e3 * _time(lambda: ops.embedding_sgd(model.target_embeds, [(b1, out["gt"], 1, 1.0)], 0.0),
                                               args.reps),
        "embedding_sgd_context_us": 1e3 * _time(lambda: ops.embedding_sgd(ctx, [(b2, out["gc_pos"], 1, 1.0),
                                                                               (neg, out["gc_neg"], 1, 1.0)], 0.0), args.reps),
    }
    model.neg_sampler.check()
    print(json.dumps({"card": _card(), "shape": {"V": V, "d": D, "B": B, "S": S}, "steps": args.steps,
                      "rounds": rounds, "kernels": kernels}))


if __name__ == "__main__":
    main()
