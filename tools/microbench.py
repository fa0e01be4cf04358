"""Kernel-level timings on the Reddit-shape workload (run on the GPU; writes out/micro_*.json).
Times each kernel alone with CUDA events, fresh random ids every iteration (table 567 MB >> L2)."""
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import graphsage_b200 as gs  # noqa: E402
from graphsage_b200 import ops  # noqa: E402

N, F, B = 232965, 602, 512
P = ops.pad_cols(F)
dev = torch.device("cuda")
torch.manual_seed(0)
table = torch.randn((N + 1, P), device=dev)
table[:, F:] = 0
table[N] = 0
NIT = 30


def timeit(fn, nit=NIT, warm=3):
    for i in range(warm):
        fn(i)
    torch.cuda.synchronize()
    evs = []
    torch.cuda._sleep(4000000)   # keep the GPU busy (~2 ms) while the host enqueues: events then see pure device time
    for i in range(nit):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn(warm + i)
        e1.record()
        evs.append((e0, e1))
    torch.cuda.synchronize()
    t = np.array([a.elapsed_time(b) for a, b in evs])
    return float(np.median(t)), float(t.min())


def id_sets(uniform=True):
    rs = np.random.RandomState(0)
    sets = []
    for i in range(NIT + 3):
        if uniform:
            s0 = rs.randint(0, N, size=B)
            s1 = rs.randint(0, N, size=B * 10)
            s2 = rs.randint(0, N, size=B * 250)
        sets.append(tuple(torch.from_numpy(x.astype(np.int32)).to(dev) for x in (s0, s1, s2)))
    return sets


res = {}
sets = id_sets()
rows = B * 11
gbytes = B * 261 * F * 4
xs = torch.empty((rows, P), device=dev)
xm = torch.empty((rows, P), device=dev)
for variant in (2, 1, 0):
    for cps in (2, 3, 4, 8):
        gs._lib.set_tuning("gather_variant", variant)
        gs._lib.set_tuning("gather_ctas_per_sm", cps)

        def run(i):
            s0, s1, s2 = sets[i]
            segs = [ops.Seg(B, 10, self_ids=s0, neigh_ids=s1, out_row0=0),
                    ops.Seg(B * 10, 25, self_ids=s1, neigh_ids=s2, out_row0=B)]
            ops.gather_mean(table[:, :F], segs, out_mean=xm, out_self=xs)
        med, mn = timeit(run)
        res["gather_mean_v%d_cps%d" % (variant, cps)] = {"ms_median": med, "ms_min": mn, "alg_GBps": gbytes / med / 1e6}
        print("gather_mean variant", variant, "ctas/sm", cps, "median ms", med, "alg GB/s", gbytes / med / 1e6, flush=True)
gs._lib.set_tuning("gather_variant", 2)
gs._lib.set_tuning("gather_ctas_per_sm", 8)

allids = [torch.cat(s) for s in sets]
outbuf = torch.empty((B * 261, P), device=dev)
for variant in (1, 0):
    gs._lib.set_tuning("gather_variant", variant)
    med, mn = timeit(lambda i: ops.gather_rows(table, allids[i], out=outbuf))
    res["gather_rows_v%d" % variant] = {"ms_median": med, "ms_min": mn, "alg_GBps_read": B * 261 * P * 4 / med / 1e6}
    print("gather_rows variant", variant, med, "read GB/s", B * 261 * P * 4 / med / 1e6, flush=True)
gs._lib.set_tuning("gather_variant", 1)
med, _ = timeit(lambda i: table.index_select(0, allids[i].long()))
res["torch_index_select"] = {"ms_median": med}
print("torch index_select", med, flush=True)

# GEMM: layer 0 shape [5632, 602] x [602,128] x2 concat
Ws, Wn = torch.randn(F, 128, device=dev), torch.randn(F, 128, device=dev)
for math in ("fp32", "tf32x3", "tf32", "bf16"):
    try:
        code = gs.aggregators._MATH_NAMES[math]
        med, mn = timeit(lambda i: ops.sage_gemm([(xs, F, Ws), (xm, F, Wn)], combine=ops.COMBINE_CONCAT, act=ops.ACT_RELU,
                                                 math=code))
        res["gemm_l0_" + math] = {"ms_median": med, "ms_min": mn, "TFLOPs": 2 * 2 * rows * F * 128 / med / 1e9}
        print("gemm", math, med, flush=True)
    except RuntimeError as e:
        print("gemm", math, "unavailable:", str(e)[:80])
med, _ = timeit(lambda i: torch.relu(torch.cat([xs[:, :F] @ Ws, xm[:, :F] @ Wn], 1)))
res["torch_gemm_l0"] = {"ms_median": med}
# fused small layer (layer 1 at bench size): [512 rows] mean over 10 of [5120, 256] -> 2 x [256,128] -> l2norm
H1 = torch.randn(B * 11, 256, device=dev)
W1s, W1n = torch.randn(256, 128, device=dev), torch.randn(256, 128, device=dev)
seg1 = ops.Seg(B, 10, self_row0=0, neigh_row0=B)
med, mn = timeit(lambda i: ops.sage_layer_small(H1, seg1, [(None, 256, W1s), (None, 256, W1n)], combine=ops.COMBINE_CONCAT,
                                                l2_normalize=True))
res["layer_small_512"] = {"ms_median": med, "ms_min": mn}
print("layer_small", med, flush=True)
packed = ops.PackedWeights()
for math in ("tf32x3", "bf16"):
    code = gs.aggregators._MATH_NAMES[math]
    med, mn = timeit(lambda i: ops.sage_gemm([(xs, F, Ws), (xm, F, Wn)], combine=ops.COMBINE_CONCAT, act=ops.ACT_RELU,
                                             math=code, packed=packed))
    res["gemm_l0_prepacked_" + math] = {"ms_median": med, "ms_min": mn}
    print("gemm prepacked", math, med, flush=True)
# sampler
adj = torch.randint(0, N, (N + 1, 128), device=dev, dtype=torch.int32)
med, _ = timeit(lambda i: ops.sample_padded(adj, sets[i][1], 25, 123, i))
res["sample_5120x25"] = {"ms_median": med}
med, _ = timeit(lambda i: ops.sample_padded(adj, sets[i][0], 10, 123, i))
res["sample_512x10"] = {"ms_median": med}
med, _ = timeit(lambda i: ops.sample_padded_khop(adj, sets[i][0], [10, 25], 123, i))
res["sample_khop_512x10x25"] = {"ms_median": med}
print(json.dumps(res, indent=1))
os.makedirs("out", exist_ok=True)
json.dump(res, open("out/micro_%s.json" % os.environ.get("MICRO_TAG", "r1"), "w"), indent=1)
