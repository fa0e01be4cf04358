"""Time full-neighbourhood inference on the GPU: gs_csr_aggregate at layer 0 and the whole
SampleAndAggregate.full_neighbor_embeddings pass against the sampled export_embeddings over every node.

    python tools/full_neighbor_bench.py [--iters 10] [--rounds 2] [--rmat-scale 18] [--out full_neighbor_bench.json]

Inputs: "community" = community_graph_csr(232,965, mean_deg=50) (Reddit's node count and density, degrees up to 2,000)
with 602 random features, fp32 and bf16; "rmat" = rmat_csr_device(--rmat-scale) (hubs far above the community cap) with
the same feature width.  Per input and op: CUDA events around --iters gs_csr_aggregate calls over all N+1 rows after
warm-up, and the algorithmic bytes over that time: every CSR entry's feature row (F elements), the output rows
(out_pitch fp32), the indices and indptr - no cache reuse credited.  The pass: a 2-layer concat model (fanouts 25, 10,
width 128 per half; mean and max-pool) timed end to end with a device synchronise, against export_embeddings of every
node on the same model, with torch.cuda.max_memory_allocated above the resident set for each.  Everything is measured
--rounds times in the one process; the card name and power limit are read in the same command."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import graphsage_b200 as gs  # noqa: E402
from graphsage_b200 import ops  # noqa: E402
from graphsage_b200.minibatch import padded_from_csr_fast  # noqa: E402
from graphsage_b200.synthetic import community_graph_csr, rmat_csr_device  # noqa: E402

F = 602


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def table(n_rows, dtype, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    t = torch.zeros((n_rows, ops.pad_cols(F)), dtype=torch.float32, device="cuda")
    t[:-1, :F] = torch.randn((n_rows - 1, F), generator=g, device="cuda")
    return t.to(dtype)[:, :F]


def kernel_time(src, indptr, indices, op, iters):
    n = indptr.numel()                               # N + 1 output rows
    out = torch.empty((n, ops.pad_cols(F)), dtype=torch.float32, device="cuda")
    for _ in range(2):
        ops.csr_aggregate(src, indptr, indices, op, out=out)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        ops.csr_aggregate(src, indptr, indices, op, out=out)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / iters
    deg = (indptr[1:] - indptr[:-1])
    entries = int(torch.clamp(deg, min=1).sum()) + 1 + (n if op == "mean_self" else 0)   # the dummy node: one entry
    nbytes = entries * F * src.element_size() + n * out.stride(0) * 4 + indices.numel() * 4 + indptr.numel() * 8
    return {"op": op, "dtype": str(src.dtype).replace("torch.", ""), "ms": ms, "gathered_rows": entries,
            "algorithmic_GB": nbytes / 1e9, "algorithmic_TB_per_s": nbytes / ms / 1e9}


def pass_times(features, indptr_h, indices_h, kind):
    n = len(indptr_h) - 1
    adj, _ = padded_from_csr_fast(indptr_h, indices_h, 128)
    adj = torch.from_numpy(adj).cuda()
    gs.set_default_math("tf32x3")
    gs.inits.manual_seed(1)
    sampler = gs.UniformNeighborSampler(adj, seed=123)
    infos = [gs.SAGEInfo("node", sampler, 25, 128), gs.SAGEInfo("node", sampler, 10, 128)]
    m = gs.SampleAndAggregate({"batch_size": 512, "dropout": 0.}, features, adj, None, infos, concat=True,
                              aggregator_type=kind)
    indptr, indices = torch.from_numpy(indptr_h).cuda(), torch.from_numpy(indices_h).cuda()
    ids = np.arange(n, dtype=np.int32)
    m.export_embeddings(ids[:4096])
    m.full_neighbor_embeddings(indptr, indices, node_ids=ids[:4096])
    res = {"aggregator": kind}
    for name, fn in (("full_neighbor_embeddings", lambda: m.full_neighbor_embeddings(indptr, indices)),
                     ("export_embeddings", lambda: m.export_embeddings(ids))):
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        res[name + "_s"] = time.perf_counter() - t0
        res[name + "_peak_MB"] = (torch.cuda.max_memory_allocated() - base) / 2**20
    res["nodes_per_s_full"] = n / res["full_neighbor_embeddings_s"]
    res["nodes_per_s_export"] = n / res["export_embeddings_s"]
    gs.set_default_math("fp32")
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--rmat-scale", type=int, default=18)
    ap.add_argument("--out", default="full_neighbor_bench.json")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "the benchmark needs a CUDA device"
    gs._lib.lib()
    res = {"card": card(), "rounds": []}
    t0 = time.perf_counter()
    ip, ix, _ = community_graph_csr(232965, mean_deg=50)
    res["community"] = {"nodes": len(ip) - 1, "entries": int(ip[-1]), "max_degree": int(np.diff(ip).max()),
                        "build_s": time.perf_counter() - t0}
    rp, rx = rmat_csr_device(a.rmat_scale)
    rdeg = (rp[1:] - rp[:-1])
    res["rmat"] = {"scale": a.rmat_scale, "nodes": rp.numel() - 1, "entries": int(rp[-1]), "max_degree": int(rdeg.max()),
                   "rows_over_256": int((rdeg > 256).sum())}
    cp, cx = torch.from_numpy(ip).cuda(), torch.from_numpy(ix).cuda()
    f32 = table(len(ip), torch.float32)
    bf = table(len(ip), torch.bfloat16)
    rt = table(rp.numel(), torch.float32, seed=1)
    for r in range(a.rounds):
        rnd = {"kernel": []}
        for src, p, x, name in ((f32, cp, cx, "community"), (bf, cp, cx, "community"), (rt, rp, rx, "rmat")):
            for op in ("mean", "max") if src.dtype == torch.float32 else ("mean",):
                k = kernel_time(src, p, x, op, a.iters)
                k["graph"] = name
                rnd["kernel"].append(k)
                print(json.dumps(k), flush=True)
        rnd["pass"] = [pass_times(f32, ip, ix, kind) for kind in ("mean", "maxpool")]
        for p_ in rnd["pass"]:
            print(json.dumps(p_), flush=True)
        res["rounds"].append(rnd)
    print(json.dumps({k: v for k, v in res.items() if k != "rounds"}))
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as fp:
        json.dump(res, fp, indent=1)


if __name__ == "__main__":
    main()
