"""Time SGDClassifier(loss="log") of the eval scripts on the GPU against the installed scikit-learn.

    python tools/eval_bench.py [--runs 2] [--skip-sklearn] [--out eval_bench.json]

Random Reddit-sized (152,410 x 256 fp64, 41 classes, one-vs-rest) and PPI-sized (44,906 x 256 fp64, 121 0/1 columns)
problems with l2-normalised rows.  Per run: the orders (gs_sgd_orders) and the SGD (gs_sgd_fit) in CUDA events, and the
host clock around a whole synchronised SGDClassifier.fit (host label and seed set-up and copies included).  scikit-learn
(SGDClassifier(loss="log_loss", max_iter=5, tol=None), n_jobs=1 and n_jobs = all host cores) runs on the same arrays when
it is importable.  The card name and power limit are read in the same command."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from graphsage_b200 import linear_model as lm  # noqa: E402


def problems():
    rs = np.random.RandomState(0)
    out = {}
    for name, n, d in [("reddit", 152410, 256), ("ppi", 44906, 256)]:
        x = rs.randn(n, d)
        x /= np.linalg.norm(x, axis=1, keepdims=True)
        if name == "reddit":
            y = rs.randint(0, 41, size=n)
            labels = np.where(y[None, :] == np.arange(41)[:, None], 1, -1)
        else:
            y = (rs.rand(n, 121) < rs.uniform(0.05, 0.6, size=121)).astype(np.int64)
            labels = np.where(y.T == 1, 1, -1)
        out[name] = (x, y, np.ascontiguousarray(labels, dtype=np.int32))
    return out


def gpu_split(x, labels):
    """(orders ms, sgd ms) in CUDA events for one fit of the problems."""
    xt, lt = torch.from_numpy(x).cuda(), torch.from_numpy(labels).cuda()
    seeds = np.random.RandomState(1).randint(0, 2 ** 31 - 1, size=labels.shape[0])
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    ev[0].record()
    orders = lm.sgd_orders(seeds, x.shape[0], "cuda")
    ev[1].record()
    lm.sgd_fit(xt, lt, orders)
    ev[2].record()
    torch.cuda.synchronize()
    return ev[0].elapsed_time(ev[1]), ev[1].elapsed_time(ev[2])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=2)
    ap.add_argument("--skip-sklearn", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("eval_bench needs a CUDA device")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    result = {"gpu": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip(), "runs": []}
    data = problems()
    for name, (x, y, labels) in data.items():        # warm-up: module load, both kernels at this shape
        gpu_split(x[:4096], np.ascontiguousarray(labels[:, :4096]))
    for r in range(args.runs):
        for name, (x, y, labels) in data.items():
            orders_ms, sgd_ms = gpu_split(x, labels)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            np.random.seed(1)
            lm.SGDClassifier().fit(x, y)
            torch.cuda.synchronize()
            fit_s = time.perf_counter() - t0
            row = {"run": r, "problem": name, "orders_ms": orders_ms, "sgd_ms": sgd_ms, "fit_s": fit_s}
            print(json.dumps(row), flush=True)
            result["runs"].append(row)
    if not args.skip_sklearn:
        try:
            from sklearn.linear_model import SGDClassifier
            from sklearn.multioutput import MultiOutputClassifier
        except ImportError:
            result["sklearn"] = "not importable"
        else:
            for r in range(args.runs):
                for name, (x, y, labels) in data.items():
                    for jobs in (1, os.cpu_count()):
                        est = SGDClassifier(loss="log_loss", max_iter=5, tol=None, n_jobs=jobs if name == "reddit" else None)
                        if name == "ppi":
                            est = MultiOutputClassifier(est, n_jobs=jobs)
                        t0 = time.perf_counter()
                        est.fit(x, y)
                        row = {"run": r, "problem": name, "sklearn_n_jobs": jobs, "sklearn_fit_s": time.perf_counter() - t0}
                        print(json.dumps(row), flush=True)
                        result["runs"].append(row)
    print(json.dumps({k: v for k, v in result.items() if k != "runs"}))
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as fp:
            json.dump(result, fp, indent=1)


if __name__ == "__main__":
    main()
