"""Time sampled-block training (SupervisedGraphsage.sampled_minibatch_train_step) on host-memory and int8 feature tables
against the device fp32 table, and the layer-0 loader (HostFeatures.gather_rows_f32, gs_host_gather_rows_f32) against the
composition it replaces: gs_host_fetch of V_0's uncached rows into a working set, then gs_gather_rows_f32 over it.

    python tools/sampled_host_bench.py [--iters 5] [--rounds 2] [--reps 20] [--out sampled_host_bench.json]

Graph and model as tools/sampled_blocks_bench.py: community_graph_csr(232,965, mean_deg=50), 602 random features, 2
layers, concat, width 128, tf32x3, 41 classes, fanouts (25, 10), batches of 512 random ids; mean and max-pool.
Cases: device fp32; host fp32 with 0 % and 50 % of the rows cached (hot_rows((indptr, indices), C), by in-degree);
device int8; host int8 with 0 % and 50 % cached.  Per case and aggregator:
  V0              |V_0| of the step's block set;
  link_rows       V_0's uncached rows (read over the host link; 0 on the device);
  link_MB         the bytes the loader asks of the link: link_rows x the 16-byte units that hold columns [0, F);
  loader_us, loader_GBps   one layer-0 load of V_0 (CUDA events over --reps calls): the fused loader for a host table,
                  ops.gather_rows_f32 for device int8 (device fp32 has none: layer 0 reads the table by id);
  compose_us, compose_GBps (host cases) gs_host_fetch of the link rows (whole rows, row_bytes each) + gs_gather_rows_f32
                  over the working set, timed alternately with the loader in the same process;
  step_ms, peak_MB   sampled_minibatch_train_step (--iters steps), peak device memory above the resident set.
The card name and power limit are read in the same command."""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import graphsage_b200 as gs  # noqa: E402
from graphsage_b200 import ops  # noqa: E402
from graphsage_b200.host_features import hot_rows  # noqa: E402
from graphsage_b200.minibatch import padded_from_csr_fast  # noqa: E402
from graphsage_b200.synthetic import community_graph_csr  # noqa: E402
from sampled_blocks_bench import BATCH, C, F, FANOUTS, MEAN_DEG, N_NODES, Timer, card, timed_steps  # noqa: E402


def build_model(kind, features, adj):
    """sampled_blocks_bench's model without a batch_size placeholder: a host table then reserves no tree-path staging."""
    gs.set_default_math("tf32x3")
    gs.inits.manual_seed(1)
    sampler = gs.UniformNeighborSampler(adj, seed=123)
    infos = [gs.SAGEInfo("node", sampler, k, 128) for k in FANOUTS]
    m = gs.SupervisedGraphsage(C, {"dropout": 0.}, features, adj, None, infos, concat=True, aggregator_type=kind,
                               learning_rate=0.01)
    gs.set_default_math("fp32")
    return m


def unit_bytes(dtype):
    """Link bytes per row of the fused loader: the 16-byte units holding columns [0, F)."""
    w = {torch.float32: 4, torch.bfloat16: 8, torch.int8: 16}[dtype]
    return (F + w - 1) // w * 16


def composition(h, v0):
    """A closure running gs_host_fetch of v0's uncached rows + gs_gather_rows_f32 over the resulting working set, and the
    bytes the fetch moves."""
    slot = h.cache_slot[v0.long()]
    miss = slot < 0
    stage = v0[miss].contiguous()
    U, Cc = stage.numel(), h.n_cached
    ws = torch.empty((Cc + 1 + U, h.ws.shape[1]), dtype=h.ws.dtype, device=h.ws.device)
    ws[:Cc + 1].copy_(h.ws[:Cc + 1])
    rows = torch.where(miss, Cc + 1 + torch.cumsum(miss.to(torch.int32), 0, dtype=torch.int32) - 1, slot)
    rows = rows.to(torch.int32).contiguous()
    count = torch.full((1,), U, dtype=torch.int32, device=v0.device)
    src = ops.I8Rows(ws, F) if h.dtype == torch.int8 else ws[:, :F]

    def run():
        ops.host_fetch(h._alias, h.row_bytes, stage, count, ws[Cc + 1:])
        return ops.gather_rows_f32(src, rows)
    return run, U * h.row_bytes


def time_calls(fn, reps):
    with Timer() as t:
        for _ in range(reps):
            fn()
    return t.ms * 1e3 / reps


def measure(case, kind, features, adj, indptr, indices, ids, labels, iters, reps):
    m = build_model(kind, features, adj)
    sampler = m.layer_infos[0].neigh_sampler
    res = {"case": case, "aggregator": kind}
    v0 = ops.csr_blocks(indptr, indices, ids, 2, fanouts=FANOUTS, seed=sampler.seed, call=sampler.counter)[0].src_ids
    res["V0"] = int(v0.numel())
    host = isinstance(features, gs.HostFeatures)
    if host:
        link = int((features.cache_slot[v0.long()] < 0).sum())
        res["link_rows"], res["link_MB"] = link, link * unit_bytes(features.dtype) / 1e6
        loader = lambda: features.gather_rows_f32(v0)                               # noqa: E731
        compose, compose_bytes = composition(features, v0)
        assert torch.equal(loader(), compose())
        for r in range(2):                                          # alternating, after the warm-up above
            res.setdefault("loader_us", []).append(time_calls(loader, reps))
            res.setdefault("compose_us", []).append(time_calls(compose, reps))
        res["loader_GBps"] = [res["link_MB"] * 1e6 / (us * 1e3) for us in res["loader_us"]]
        res["compose_MB"] = compose_bytes / 1e6
        res["compose_GBps"] = [compose_bytes / (us * 1e3) for us in res["compose_us"]]
        del compose
    elif features.dtype == torch.int8:
        res["link_rows"], res["link_MB"] = 0, 0.
        ops.gather_rows_f32(features, v0)
        res["loader_us"] = [time_calls(lambda: ops.gather_rows_f32(features, v0), reps)]
    else:
        res["link_rows"], res["link_MB"], res["loader_us"] = 0, 0., None
    m.sampled_minibatch_train_step(indptr, indices, ids, labels)                  # warm-up: Adam state
    res["step_ms"], res["peak_MB"] = timed_steps(lambda: m.sampled_minibatch_train_step(indptr, indices, ids, labels),
                                                 iters)
    del m
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default="sampled_host_bench.json")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "the benchmark needs a CUDA device"
    gs._lib.lib()
    res = {"card": card(), "rounds": [[] for _ in range(a.rounds)]}
    print(json.dumps({"card": res["card"]}), flush=True)
    ip, ix, _ = community_graph_csr(N_NODES, mean_deg=MEAN_DEG)
    n = len(ip) - 1
    res["graph"] = {"nodes": n, "entries": int(ip[-1]), "features": F}
    print(json.dumps(res["graph"]), flush=True)
    g = torch.Generator(device="cuda").manual_seed(0)
    t = torch.zeros((n + 1, ops.pad_cols(F)), dtype=torch.float32, device="cuda")
    t[:-1, :F] = torch.randn((n, F), generator=g, device="cuda")
    dev_f32 = t[:, :F]
    host_f32 = dev_f32.cpu()
    dev_i8 = gs.Int8Features(dev_f32)
    host_i8 = gs.Int8Features(host_f32)
    hot = hot_rows((ip, ix), n // 2)
    tables = [("device fp32", lambda: dev_f32), ("host fp32 0%", lambda: gs.HostFeatures(host_f32)),
              ("host fp32 50%", lambda: gs.HostFeatures(host_f32, cache_ids=hot)), ("device int8", lambda: dev_i8),
              ("host int8 0%", lambda: gs.HostFeatures(host_i8)),
              ("host int8 50%", lambda: gs.HostFeatures(host_i8, cache_ids=hot))]
    adj = torch.from_numpy(padded_from_csr_fast(ip, ix, 128)[0]).cuda()
    indptr, indices = torch.from_numpy(ip).cuda(), torch.from_numpy(ix).cuda()
    rs = np.random.RandomState(0)
    for r in range(a.rounds):
        for case, make in tables:
            features = make()
            for kind in ("mean", "maxpool"):
                ids = torch.from_numpy(rs.choice(n, BATCH, replace=False).astype(np.int32)).cuda()
                labels = torch.zeros((BATCH, C), device="cuda")
                labels[torch.arange(BATCH, device="cuda"), torch.from_numpy(rs.randint(0, C, BATCH)).cuda()] = 1.0
                out = dict(round=r, **measure(case, kind, features, adj, indptr, indices, ids, labels, a.iters, a.reps))
                print(json.dumps(out), flush=True)
                res["rounds"][r].append(out)
            if isinstance(features, gs.HostFeatures):
                features.close()
            del features
            torch.cuda.empty_cache()
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as fp:
        json.dump(res, fp, indent=1)


if __name__ == "__main__":
    main()
