"""Time node2vec's biased walk (gs_random_walks_biased) against the uniform walk (gs_random_walks) on the GPU.

    python tools/biased_walk_bench.py [--iters 10] [--out biased_walk_bench.json]

Inputs: "reddit" = community_graph_csr(232,965, mean_deg=50) walked from 152,410 starts (the size of Reddit's walks
file), and "toy-ppi" = the toy-ppi slice's train subgraph walked from its train nodes; W = 50 walks per start, L = 5.
Per input and (p, q) in (1, 1), (0.25, 4), (4, 0.25), (0.25, 0.25), plus (0.25, 4) at L = 33 on reddit:
  - kernel_ms: CUDA events around the walk entry alone (walk kernel + CUB scan), the row sort prepared beforehand;
  - call_ms:   CUDA events around the whole ops.random_walks call (sort given, walk, scan, read-back of P, emit);
  - sort_ms:   CUDA events around ops.csr_sort_rows (start-up work, once per graph);
  walks/s and pairs/s over call_ms, and, from the oracle on a sample of 1,000 starts, the mean rejection attempts per
  move after the first and the share of those moves that fell back to the inverse-CDF draw.
"uniform" is gs_random_walks itself.  Each timing is the median over --iters calls after two warm-up calls.  The card's
name, power limit and max SM clock are read in the same command."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

from graphsage_b200 import _lib, ops  # noqa: E402
from graphsage_b200.graph import to_csr  # noqa: E402
from graphsage_b200.synthetic import community_graph_csr  # noqa: E402
from oracle import biased_walks as bw  # noqa: E402

W = 50
PQ = [(1.0, 1.0), (0.25, 4.0), (4.0, 0.25), (0.25, 0.25)]


def timed(fn, iters):
    fn()
    fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(iters):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1))
    return float(np.median(ms))


def run(name, indptr, indices, starts, L, pq, iters, srt):
    lib = _lib.lib()
    ip, ix, st = (torch.from_numpy(indptr).cuda(), torch.from_numpy(indices).cuda(), torch.from_numpy(starts).cuda())
    n = len(starts)
    nbytes = lib.gs_random_walks_workspace_bytes(n, W, L)
    ws = torch.empty((nbytes,), dtype=torch.uint8, device="cuda")
    n_pairs = torch.empty((1,), dtype=torch.int64, device="cuda")
    s = _lib.stream_ptr()
    if pq is None:
        kernel = lambda: _lib.check(lib.gs_random_walks(ip.data_ptr(), ix.data_ptr(), len(indptr) - 1, st.data_ptr(), n, W,
                                                        L, 123, 0, 0, ws.data_ptr(), nbytes, n_pairs.data_ptr(), s))
        call = lambda: ops.random_walks(ip, ix, st, W, L, 123, 0)
    else:
        p, q = pq
        kernel = lambda: _lib.check(lib.gs_random_walks_biased(
            ip.data_ptr(), ix.data_ptr(), srt.data_ptr(), len(indptr) - 1, st.data_ptr(), n, W, L, p, q, 123, 0, 0,
            ws.data_ptr(), nbytes, n_pairs.data_ptr(), s))
        call = lambda: ops.random_walks(ip, ix, st, W, L, 123, 0, p=p, q=q, sorted_indices=srt)
    kernel_ms = timed(kernel, iters)
    call_ms = timed(call, iters)
    P = len(call())
    row = {"graph": name, "p": None if pq is None else pq[0], "q": None if pq is None else pq[1], "L": L,
           "walks": n * W, "pairs": P, "kernel_ms": kernel_ms, "call_ms": call_ms,
           "walks_per_s": n * W / call_ms * 1e3, "pairs_per_s": P / call_ms * 1e3}
    if pq is not None and pq != (1.0, 1.0):
        sample = starts[np.random.RandomState(1).permutation(n)[:1000]]
        _, stats = bw.biased_random_walks(indptr, indices, sample, W, L, pq[0], pq[1], 123, stats=True)
        row["mean_attempts_per_move"] = stats["attempts"] / max(stats["steps"], 1)
        row["fallback_rate"] = stats["fallbacks"] / max(stats["steps"], 1)
    print(json.dumps(row), flush=True)
    del ws
    return row


def toy_ppi():
    from make_walks_golden import toy_graph
    G = toy_graph()
    train = [u for u in G.nodes() if not G.node[u]["val"] and not G.node[u]["test"]]
    H = G.subgraph(train)
    pos = {u: i for i, u in enumerate(H.nodes())}
    csr = to_csr(H, pos)
    return csr["indptr"].astype(np.int64), csr["indices"].astype(np.int32), np.array([pos[u] for u in train], np.int32)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("biased_walk_bench needs a CUDA device")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(smi, flush=True)
    result = {"gpu": torch.cuda.get_device_name(0), "nvidia_smi": smi, "W": W, "rows": [], "sort_ms": {}}
    indptr, indices, _ = community_graph_csr(232965, mean_deg=50, seed=123)
    graphs = [("reddit", indptr, indices, np.random.RandomState(0).permutation(232965)[:152410].astype(np.int32)),
              ("toy-ppi",) + toy_ppi()]
    for name, indptr, indices, starts in graphs:
        ip, ix = torch.from_numpy(indptr).cuda(), torch.from_numpy(indices).cuda()
        result["sort_ms"][name] = timed(lambda: ops.csr_sort_rows(ip, ix), args.iters)
        srt = ops.csr_sort_rows(ip, ix)
        result["rows"].append(run(name, indptr, indices, starts, 5, None, args.iters, srt))
        for pq in PQ:
            result["rows"].append(run(name, indptr, indices, starts, 5, pq, args.iters, srt))
        if name == "reddit":
            result["rows"].append(run(name, indptr, indices, starts, 33, None, args.iters, srt))
            result["rows"].append(run(name, indptr, indices, starts, 33, (0.25, 4.0), args.iters, srt))
    print(json.dumps({"gpu": result["gpu"], "nvidia_smi": smi, "sort_ms": result["sort_ms"]}))
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as fp:
            json.dump(result, fp, indent=1)


if __name__ == "__main__":
    main()
