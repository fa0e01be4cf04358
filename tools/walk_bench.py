"""Time the random-walk pairs (gs_random_walks + gs_random_walks_emit) on the GPU and the host walker they replace.

    python tools/walk_bench.py [--iters 20] [--out walk_bench.json]

Inputs: "reddit" = community_graph_csr(232,965, mean_deg=50) with 152,410 starts x 50 walks, L = 5 (the size of
Reddit's walks file); "50k" = a 50,000-node graph of the same density with 2,000 starts, the size the host walker is
timed at.  Per input: CUDA events around gs_random_walks (walk kernel + CUB scan) and gs_random_walks_emit over --iters
calls after warm-up, walks/s and pairs/s, and the bytes the algorithm moves, computed from shapes:
  per executed step one 32-B sector for the indptr pair and one for the indices entry (random reads); the visited ids
  (4 B per step, written and read), the counts (1 B per walk, written and read twice), the offsets (8 B per walk,
  written and read), the starts (4 B per walk, read twice) and the [P, 2] int32 output (8 B per pair).
The host side, in the same process: utils.run_random_walks on the 50k graph as microseconds per walk, and the stages of
`python -m graphsage_b200.utils` after the JSON parse on the 50k graph walked from every node: to_csr, the device walk
with its copies back and name mapping, and the text formatting.  The card name and power limit are read in the same
command."""
import argparse
import json
import os
import random
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from graphsage_b200 import _lib, ops, utils  # noqa: E402
from graphsage_b200.graph import Graph, to_csr  # noqa: E402
from graphsage_b200.synthetic import community_graph_csr  # noqa: E402

L, W = 5, 50
HBM_TBS = 3.35          # H100 SXM data-sheet HBM3 bandwidth, TB/s


def device_times(indptr, indices, starts, iters):
    """(walk + scan ms, emit ms, pairs, executed steps) per call, CUDA events, after one warm-up call."""
    lib = _lib.lib()
    n = starts.numel()
    nbytes = lib.gs_random_walks_workspace_bytes(n, W, L)
    ws = torch.empty((nbytes,), dtype=torch.uint8, device="cuda")
    n_pairs = torch.empty((1,), dtype=torch.int64, device="cuda")
    st = _lib.stream_ptr()

    def walk():
        _lib.check(lib.gs_random_walks(indptr.data_ptr(), indices.data_ptr(), indptr.numel() - 1, starts.data_ptr(), n, W,
                                       L, 123, 0, 0, ws.data_ptr(), nbytes, n_pairs.data_ptr(), st))

    walk()
    P = int(n_pairs.item())
    out = torch.empty((P, 2), dtype=torch.int32, device="cuda")

    def emit():
        _lib.check(lib.gs_random_walks_emit(starts.data_ptr(), n, W, L, ws.data_ptr(), nbytes, out.data_ptr(), st))

    emit()
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    walk_ms = emit_ms = 0.0
    for _ in range(iters):
        ev[0].record()
        walk()
        ev[1].record()
        emit()
        ev[2].record()
        torch.cuda.synchronize()
        walk_ms += ev[0].elapsed_time(ev[1])
        emit_ms += ev[1].elapsed_time(ev[2])
    # executed steps: every walk from a start with neighbours takes L - 1 steps on these undirected graphs
    deg = (indptr[starts.long() + 1] - indptr[starts.long()]).cpu().numpy()
    steps = int(np.count_nonzero(deg > 0)) * W * (L - 1)
    return walk_ms / iters, emit_ms / iters, P, steps


def algorithmic_bytes(walks, steps, pairs):
    return steps * 64 + steps * 4 * 2 + walks * (1 * 3 + 8 * 2 + 4 * 2) + pairs * 8


def graph_from_csr(indptr, indices):
    G = Graph()
    for u in range(len(indptr) - 1):
        G.add_node(u, val=False, test=False)
    for u in range(len(indptr) - 1):
        for v in indices[indptr[u]:indptr[u + 1]].tolist():
            if v > u:
                G.add_edge(u, v)
    return G


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("walk_bench needs a CUDA device")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    result = {"gpu": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip(), "L": L, "W": W, "inputs": {}}
    print(result["nvidia_smi"], flush=True)
    graphs = {}
    for name, n, n_starts in [("reddit", 232965, 152410), ("50k", 50000, 2000)]:
        indptr, indices, _ = community_graph_csr(n, mean_deg=50, seed=123)
        graphs[name] = (indptr, indices)
        starts = np.random.RandomState(0).permutation(n)[:n_starts].astype(np.int32)
        ip, ix, st = (torch.from_numpy(indptr).cuda(), torch.from_numpy(indices).cuda(), torch.from_numpy(starts).cuda())
        walk_ms, emit_ms, P, steps = device_times(ip, ix, st, args.iters)
        walks = n_starts * W
        total_s = (walk_ms + emit_ms) / 1e3
        nbytes = algorithmic_bytes(walks, steps, P)
        row = {"nodes": n, "mean_row_length": float(indptr[-1]) / n, "starts": n_starts, "walks": walks, "pairs": P,
               "walk_scan_ms": walk_ms, "emit_ms": emit_ms, "walks_per_s": walks / total_s, "pairs_per_s": P / total_s,
               "algorithmic_bytes": nbytes, "implied_TB_per_s": nbytes / total_s / 1e12,
               "share_of_hbm_datasheet": nbytes / total_s / 1e12 / HBM_TBS}
        result["inputs"][name] = row
        print(name, json.dumps(row), flush=True)

    # host walker, same 50k graph and starts
    indptr, indices = graphs["50k"]
    t0 = time.perf_counter()
    G = graph_from_csr(indptr, indices)
    build_s = time.perf_counter() - t0
    starts = np.random.RandomState(0).permutation(50000)[:2000].tolist()
    t0 = time.perf_counter()
    pairs = utils.run_random_walks(G, starts, num_walks=W, rng=random.Random(0))
    host_s = time.perf_counter() - t0
    result["host_run_random_walks"] = {"walks": 2000 * W, "seconds": host_s, "us_per_walk": host_s / (2000 * W) * 1e6,
                                       "pairs": len(pairs), "graph_build_s": build_s}
    print("host", json.dumps(result["host_run_random_walks"]), flush=True)

    # the entry point's stages after the JSON parse, every node of the 50k graph a start
    nodes = G.nodes()
    utils.run_random_walks_device(G, nodes[:100])                       # warm-up
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    to_csr(G, {n: i for i, n in enumerate(nodes)})
    csr_s = time.perf_counter() - t0
    t0 = time.perf_counter()
    pairs = utils.run_random_walks_device(G, nodes)                      # to_csr again, upload, walk, copies back, names
    device_s = time.perf_counter() - t0 - csr_s
    t0 = time.perf_counter()
    text = utils.format_walks(pairs)
    fmt_s = time.perf_counter() - t0
    result["entry_point_50k_all_nodes"] = {"starts": len(nodes), "pairs": len(pairs), "to_csr_s": csr_s,
                                           "device_walk_and_copies_s": device_s, "format_s": fmt_s,
                                           "text_bytes": len(text)}
    print("entry", json.dumps(result["entry_point_50k_all_nodes"]), flush=True)
    print(json.dumps({k: v for k, v in result.items() if k != "inputs"}))
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as fp:
            json.dump(result, fp, indent=1)


if __name__ == "__main__":
    main()
