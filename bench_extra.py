"""bench.py's two auxiliary workloads (BASELINE.json configs[3] and configs[4]); `python bench.py --workload unsup|rmat`.
They print one JSON line each (rank 0) in the same spirit as the contract line, but they are NOT the contract line: the
driver's runs use the default workload."""
import json
import os
import time

import numpy as np
import torch

from bench import BATCH, DIM, F, FANOUT, MAX_DEG, N_NODES, ClockSampler


def _sync(dist, dev):
    if dist is not None:
        dist.barrier()
    torch.cuda.synchronize(dev)


def _max_over_ranks(dist, dev, x):
    if dist is None:
        return x
    t = torch.tensor([x], dtype=torch.float64, device=dev)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())


def run_unsup(args, g, rank, world, local_rank, dist, dev):
    """configs[3]: unsupervised SampleAndAggregate + negative sampling (reference graphsage/models.py:332-405), one TRAINING
    step = 3 passes of the hot path (batch1, batch2, 20 shared negatives: 1044 seeds x 261 rows = 272,484 rows) + xent loss
    + backward + gradient all-reduce + clipped Adam; node-partitioned features (replicas as in the default workload)."""
    import graphsage_b200 as gs
    from graphsage_b200 import parallel
    gs.set_default_math(args.math)
    bounds = parallel.community_bounds(g["comm"], world) if world > 1 else [0, N_NODES]
    lo, hi = bounds[rank], bounds[rank + 1]
    cache_rows = int(os.environ.get("GS_HALO_CACHE_ROWS", str(parallel.default_cache_rows(N_NODES, world))))
    hot = parallel.hot_remote_rows(g["adj"], N_NODES, world, rank, cache_rows, row_start=bounds)
    shard = parallel.ShardedFeatures(g["features"][lo:hi], N_NODES, row_start=bounds, replica_ids=hot,
                                     replica_rows=g["features"][hot])
    adj_dev = torch.from_numpy(g["adj"]).to(dev)
    sampler = gs.UniformNeighborSampler(adj_dev, seed=123)
    infos = [gs.SAGEInfo("node", sampler, FANOUT[0], DIM), gs.SAGEInfo("node", sampler, FANOUT[1], DIM)]
    model = gs.UnsupervisedGraphsage({"batch_size": BATCH, "dropout": 0.}, shard, adj_dev, np.maximum(g["deg"], 1.0), infos,
                                     concat=True, aggregator_type="mean", neg_sample_size=20, learning_rate=1e-5,
                                     device=dev, distributed=world > 1, seed=123 + rank)
    rs = np.random.RandomState(2000 + rank)
    total = args.warmup + args.steps
    b1 = rs.randint(lo, hi, size=(total, BATCH)).astype(np.int32)
    b2 = g["adj"][b1, rs.randint(0, MAX_DEG, size=(total, BATCH))].astype(np.int32)      # a context node = a sampled neighbour
    b2 = np.where(b2 >= N_NODES, b1, b2)
    b1d, b2d = torch.from_numpy(b1).to(dev), torch.from_numpy(b2).to(dev)
    for i in range(args.warmup):
        model.train_step(b1d[i], b2d[i])
    _sync(dist, dev)
    clocks = ClockSampler(local_rank)
    clocks.start()
    l0 = gs.ops.LAUNCHES
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    losses = []
    for i in range(args.steps):
        losses.append(model.train_step(b1d[args.warmup + i], b2d[args.warmup + i]))
    e1.record()
    _sync(dist, dev)
    ms = _max_over_ranks(dist, dev, e0.elapsed_time(e1))
    clk = clocks.summary()
    launches = gs.ops.LAUNCHES - l0
    loss_first, loss_last = float(losses[0]), float(losses[-1])
    mrr = float(model.mrr())
    # weights must be identical on every rank
    flat = torch.cat([p.detach().reshape(-1) for p in model.parameters()])
    same = True
    if dist is not None:
        ref = flat.clone()
        dist.broadcast(ref, src=0)
        same = bool(torch.equal(ref, flat))
        t = torch.tensor([1.0 if same else 0.0], device=dev)
        dist.all_reduce(t, op=dist.ReduceOp.MIN)
        same = bool(t.item() == 1.0)
    rho = shard.remote_fraction(torch.from_numpy(b1[0]).to(dev))
    _sync(dist, dev)
    shard.close()
    if rank != 0:
        return
    rows_per_step = (2 * BATCH + 20) * 261
    print(json.dumps({
        "metric": "training_seed_nodes_per_sec", "workload": "configs[3]: unsupervised GraphSAGE training step "
        "(reddit-shape synthetic, graphsage_mean, 2-hop 25x10, batch %d pairs + 20 negatives), node-partitioned x%d, data parallel"
        % (BATCH, world), "value": world * (2 * BATCH + 20) * args.steps / (ms * 1e-3), "unit": "nodes/s",
        "edge_pairs_per_sec": world * BATCH * args.steps / (ms * 1e-3), "gathered_rows_per_sec": world * rows_per_step * args.steps / (ms * 1e-3),
        "n_gpus": world, "steps": args.steps, "warmup": args.warmup, "ms_per_step": ms / args.steps, "higher_is_better": True,
        "scaling": "weak", "dtype": "f32", "data": "synthetic", "rows_gathered_per_step_per_gpu": rows_per_step,
        "allreduce_bytes_per_step": model.last_allreduce_bytes, "weights_identical_across_ranks": same,
        "loss_first": loss_first, "loss_last": loss_last, "mrr_last": mrr, "gpu_launches": launches, "clocks": clk,
        "replica_rows_per_gpu": int(len(hot)),
        "note": "forward through the library's kernels (fused gather+mean over the partitioned table, wgmma GEMMs), backward "
                "= autograd with library GEMMs, eager launches (no CUDA graph): the step is launch-bound, not HBM-bound"}))


def run_train(args, g, rank, world, local_rank, dist, dev):
    """SURVEY 8f row 1: the SUPERVISED training step (reference graphsage/supervised_models.py:91-126): forward through the
    kernels, cross-entropy over 41 classes, backward (autograd formulas with library GEMMs), gradients clipped to +-5, Adam.
    One step = one 512-seed batch; the table is replicated (world == 1) - this is the training-throughput number that sits
    beside the CPU port's forward+backward."""
    import graphsage_b200 as gs
    gs.set_default_math(args.math)
    n_classes = 41
    table = torch.zeros((N_NODES + 1, gs.ops.pad_cols(F)), dtype=torch.float32, device=dev)
    table[:, :F] = torch.from_numpy(g["features"]).to(dev)
    adj_dev = torch.from_numpy(g["adj"]).to(dev)

    def make_model(features, identity_dim=0):
        sampler = gs.UniformNeighborSampler(adj_dev, seed=123)
        infos = [gs.SAGEInfo("node", sampler, FANOUT[0], DIM), gs.SAGEInfo("node", sampler, FANOUT[1], DIM)]
        return gs.SupervisedGraphsage(n_classes, {"batch_size": BATCH, "dropout": 0.}, features, adj_dev, None, infos,
                                      concat=True, aggregator_type="mean", sigmoid_loss=False, learning_rate=0.01, device=dev,
                                      distributed=world > 1, identity_dim=identity_dim)

    model = make_model(table[:, :F])
    rs = np.random.RandomState(4000 + rank)
    total = args.warmup + args.steps
    seeds = torch.from_numpy(rs.randint(0, N_NODES, size=(total, BATCH)).astype(np.int32)).to(dev)
    labels = torch.nn.functional.one_hot(torch.from_numpy(g["comm"][seeds.cpu().numpy().reshape(-1)].astype(np.int64)),
                                         n_classes).float().reshape(total, BATCH, n_classes).to(dev)   # label = community
    ms, losses, launches = _timed_train_steps(model, seeds, labels, args, dist, dev)
    identity = None
    if getattr(args, "identity_dim", 0) > 0:
        del model
        identity = _identity_train(args, make_model(None if args.featureless else table[:, :F], args.identity_dim), seeds,
                                   labels, ms, dist, dev)
    if rank != 0:
        return
    if identity is not None:
        print(json.dumps(identity))
        return
    print(json.dumps({
        "metric": "training_seed_nodes_per_sec", "workload": "supervised graphsage_mean training step (fwd + bwd + clipped Adam), "
        "reddit-shape synthetic, 2-hop 25x10, batch %d, 41 classes (label = community)" % BATCH,
        "value": world * BATCH * args.steps / (ms * 1e-3), "unit": "nodes/s", "n_gpus": world, "steps": args.steps,
        "warmup": args.warmup, "ms_per_step": ms / args.steps, "higher_is_better": True, "dtype": "f32", "data": "synthetic",
        "loss_first": float(losses[0]), "loss_last": float(losses[-1]), "gpu_launches": launches,
        "note": "forward = the library's kernels, backward = autograd formulas with library (cuBLAS) GEMMs; eager launches, no CUDA graph"}))


def _timed_train_steps(model, seeds, labels, args, dist, dev):
    """args.warmup untimed, then args.steps timed train_step calls; (ms per step summed over the region, losses, launches)."""
    import graphsage_b200 as gs
    for i in range(args.warmup):
        model.train_step(seeds[i], labels[i])
    _sync(dist, dev)
    l0 = gs.ops.LAUNCHES
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    losses = []
    for i in range(args.steps):
        losses.append(model.train_step(seeds[args.warmup + i], labels[args.warmup + i]))
    e1.record()
    _sync(dist, dev)
    return _max_over_ranks(dist, dev, e0.elapsed_time(e1)), losses, gs.ops.LAUNCHES - l0


def _identity_train(args, model, seeds, labels, ms_base, dist, dev):
    """The same supervised step with a trainable [N+1, D] node-embedding table (identity_dim = D; reference
    supervised_models.py:51-62), plus the two costs the table adds on their own: the embedding-gradient kernel
    (gs_embedding_grad, on the layer-0 lists of a real step) and the dense Adam update of the [N+1, D] table."""
    from graphsage_b200 import ops, supervised_models as sm
    ms, losses, launches = _timed_train_steps(model, seeds, labels, args, dist, dev)
    D, n_rows = model.embeds.shape[1], model.embeds.shape[0]
    # the layer-0 lists of one more step, replayed through the kernel alone
    seen = {}
    real = sm._embedding_grad

    def keep(emb_shape, lists, sites=None):
        seen["lists"] = lists
        return real(emb_shape, lists, sites)

    sm._embedding_grad = keep
    try:
        model.train_step(seeds[0], labels[0])
    finally:
        sm._embedding_grad = real
    lists = seen["lists"]
    contributions = sum(int(ids.numel()) for ids, _, _, _ in lists)
    out = torch.empty((n_rows, D), dtype=torch.float32, device=dev)
    reps = 20
    for _ in range(3):
        ops.embedding_grad(lists, n_rows, D, out=out)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        ops.embedding_grad(lists, n_rows, D, out=out)
    e1.record()
    torch.cuda.synchronize(dev)
    kernel_us = e0.elapsed_time(e1) * 1e3 / reps
    kernel_bytes = contributions * (4 + 4 * D) + n_rows * D * 4     # ids + one gradient row per contribution + dense output
    # dense Adam over the table alone (reads param, grad, m, v; writes param, m, v)
    emb = model.embeds
    emb.grad = out.clone()
    opt = torch.optim.Adam([emb], lr=0.01)
    for _ in range(3):
        opt.step()
    e0.record()
    for _ in range(reps):
        opt.step()
    e1.record()
    torch.cuda.synchronize(dev)
    adam_us = e0.elapsed_time(e1) * 1e3 / reps
    F_in = model.features.shape[1] - D
    return {
        "metric": "training_seed_nodes_per_sec", "workload": "supervised graphsage_mean training step (fwd + bwd + clipped Adam) "
        "with a trainable [N+1, %d] node-embedding table%s, reddit-shape synthetic, 2-hop 25x10, batch %d, 41 classes"
        % (D, " and no features" if F_in == 0 else " before %d feature columns" % F_in, BATCH),
        "value": BATCH * args.steps / (ms * 1e-3), "unit": "nodes/s", "n_gpus": 1, "steps": args.steps,
        "warmup": args.warmup, "ms_per_step": ms / args.steps, "ms_per_step_without_embeddings": ms_base / args.steps,
        "identity_dim": D, "features": F_in, "higher_is_better": True, "dtype": "f32", "data": "synthetic",
        "loss_first": float(losses[0]), "loss_last": float(losses[-1]), "gpu_launches": launches,
        "embedding_grad": {"us": kernel_us, "contributions": contributions, "lists": len(lists), "algorithmic_bytes": kernel_bytes,
                           "GB_per_s": kernel_bytes / (kernel_us * 1e-6) / 1e9},
        "adam_embeddings": {"us": adam_us, "bytes_per_tensor": n_rows * D * 4, "algorithmic_bytes": 7 * n_rows * D * 4,
                            "GB_per_s": 7 * n_rows * D * 4 / (adam_us * 1e-6) / 1e9},
        "note": "the without-embeddings step runs first in the same process on the same seeds; embedding_grad = one call of "
                "the library's deterministic scatter kernel on the layer-0 lists of a real step; adam_embeddings = "
                "torch.optim.Adam.step over the [N+1, D] table view alone"}


def run_rmat(args, rank, world, local_rank, dist, dev):
    """configs[4]: R-MAT graph (a, b, c, d = 0.57, 0.19, 0.19, 0.05; --rmat-scale / --rmat-nodes; BASELINE: scale 27 trimmed to
    10^8 nodes, ~20 entries per node), F = 256, graphsage_mean 2-hop 25x10, batch 512.  The graph is generated ON the GPU
    as CSR (gs_rmat_degrees / gs_rmat_fill; every GPU holds the whole CSR, 8.8 GB at full size), sampled per node from the
    CSR (gs_sample_csr - no padded table exists at this size), features node-partitioned over the GPUs in equal id ranges
    (R-MAT has no locality) with the highest-in-degree remote rows replicated, halo rows pulled over NVLink by the gather."""
    import graphsage_b200 as gs
    from graphsage_b200 import ops, parallel
    from graphsage_b200.synthetic import rmat_csr_device
    gs.set_default_math(args.math)
    Fr = 256
    n = args.rmat_nodes if args.rmat_nodes else 1 << args.rmat_scale
    t0 = time.perf_counter()
    indptr, indices = rmat_csr_device(args.rmat_scale, n, 20.0, seed=123, device=dev)
    torch.cuda.synchronize(dev)
    t_gen = time.perf_counter() - t0
    m = int(indices.numel())
    bounds = parallel.uniform_bounds(n, world)
    lo, hi = bounds[rank], bounds[rank + 1]
    cache_frac = float(os.environ.get("GS_HALO_CACHE_FRAC", "0.02"))
    hot = parallel.hot_remote_rows_csr(indices, n, world, rank, int(cache_frac * n), row_start=bounds)
    shard = parallel.ShardedFeatures(None, n, row_start=bounds, replica_ids=hot, n_features=Fr)
    gen = torch.Generator(device=dev)
    gen.manual_seed(1234 + rank)
    for i in range(0, hi - lo, 1 << 20):                       # features ~ N(0, 1), produced on the device shard by shard
        j = min(hi - lo, i + (1 << 20))
        shard.local[i:j, :Fr] = torch.randn((j - i, Fr), generator=gen, device=dev)
    t1 = time.perf_counter()
    shard.fill_replicas()
    t_rep = time.perf_counter() - t1
    sampler = gs.CSRNeighborSampler(indptr, indices, seed=123)
    infos = [gs.SAGEInfo("node", sampler, FANOUT[0], DIM), gs.SAGEInfo("node", sampler, FANOUT[1], DIM)]
    model = gs.SampleAndAggregate({"batch_size": BATCH, "dropout": 0.}, shard, None, None, infos, concat=True,
                                  aggregator_type="mean", device=dev)
    R = args.repeats if args.repeats > 0 else int(min(100, max(5, np.ceil(2000.0 / max(args.steps, 1)))))
    rs = np.random.RandomState(3000 + rank)
    total = args.warmup + args.steps * R
    seeds = torch.from_numpy(rs.randint(lo, hi, size=(total, BATCH)).astype(np.int32)).to(dev)
    model.forward(seeds[0])
    pipe = model.pipelined(BATCH, normalize=True, depth=args.depth)
    cur = torch.cuda.current_stream(dev)
    for i in range(args.warmup):
        pipe.submit_device(seeds[i])
    pipe.synchronize()
    _sync(dist, dev)
    clocks = ClockSampler(local_rank)
    clocks.start()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    regions = []
    for rep in range(R):
        base = args.warmup + rep * args.steps
        for c in pipe.computes:
            c.wait_stream(cur)
        e0.record(cur)
        for c in pipe.computes:
            c.wait_event(e0)
        for i in range(args.steps):
            pipe.submit_device(seeds[base + i])
        for c in pipe.computes:
            cur.wait_stream(c)
        e1.record(cur)
        pipe.synchronize()
        _sync(dist, dev)
        regions.append(_max_over_ranks(dist, dev, e0.elapsed_time(e1)))
    clk = clocks.summary()
    launches = pipe.runners[0].launches_per_replay
    pipe.close()
    probe = "gather_mean/%d" % (BATCH * 11)
    runner = model.graphed(BATCH, normalize=True, probe=probe)
    for i in range(min(args.warmup, 5)):
        runner(seeds[i])
    _sync(dist, dev)
    n_probe = args.steps * min(R, 5)
    pev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(n_probe)]
    for i in range(n_probe):
        runner(seeds[args.warmup + i], probe_events=pev[i])
    _sync(dist, dev)
    runner.close()
    kernel_ms = _max_over_ranks(dist, dev, float(np.mean([a.elapsed_time(b) for a, b in pev])))
    smp, _ = model.sample(seeds[1], infos)
    allids = torch.cat(smp)
    rho0 = _max_over_ranks(dist, dev, shard.remote_fraction(allids, use_replicas=False))
    rho = _max_over_ranks(dist, dev, shard.remote_fraction(allids))
    deg_max = int((indptr[1:] - indptr[:-1]).max().item())
    _sync(dist, dev)
    shard.close()
    if rank != 0:
        return
    ms = float(np.median(regions))
    rows = BATCH * 261
    gbytes = rows * Fr * 4
    peak = 6572.5
    pk = os.path.join(os.path.dirname(os.path.abspath(__file__)), "MEASURED_PEAKS.json")
    if os.path.exists(pk):
        peak = float(json.load(open(pk))["hbm_gbs"])
    print(json.dumps({
        "metric": "seed_nodes_per_sec", "workload": "configs[4]: R-MAT scale %d, %d nodes, %d CSR entries (%.1f per node, max degree %d), "
        "F=%d fp32, graphsage_mean 2-hop 25x10 batch %d, CSR per-node sampler, features node-partitioned x%d"
        % (args.rmat_scale, n, m, m / float(n), deg_max, Fr, BATCH, world),
        "value": world * BATCH * args.steps / (ms * 1e-3), "unit": "nodes/s", "n_gpus": world, "steps": args.steps,
        "warmup": args.warmup, "ms_per_step": ms / args.steps, "region_ms": {"median": ms, "min": float(min(regions)), "max": float(max(regions)), "n": len(regions)},
        "higher_is_better": True, "scaling": "weak", "dtype": "f32", "data": "synthetic", "gpu_launches": launches * args.steps,
        "launches_per_step": launches, "clocks": clk,
        "graph": {"generated_on": "device (gs_rmat_degrees + prefix sum + gs_rmat_fill)", "seconds": t_gen, "csr_bytes_per_gpu": m * 4 + (n + 1) * 8,
                  "feature_bytes_per_gpu": (hi - lo + 1 + len(hot)) * ops.pad_cols(Fr) * 4, "replica_fill_seconds": t_rep},
        "partition": {"kind": "equal contiguous id ranges (ids scrambled by the generator)", "remote_row_fraction_by_partition": rho0,
                      "remote_row_fraction_after_replicas": rho, "replica_rows_per_gpu": int(len(hot)),
                      "replica_fraction_of_table": len(hot) / float(n)},
        "gather_kernel_ms": kernel_ms, "gather_algorithmic_bytes": gbytes,
        "roofline": {"bound": "nvlink" if world > 1 and rho > 0.15 else "hbm", "kernel": "gather_mean (layer 0, hops 0+1) over the partitioned table",
                     "achieved_GBps_algorithmic": gbytes / (kernel_ms * 1e-3) / 1e9, "hbm_peak_GBps": peak,
                     "frac_of_hbm_peak": gbytes / (kernel_ms * 1e-3) / 1e9 / peak,
                     "nvlink_GBps_per_gpu": rho * gbytes / (kernel_ms * 1e-3) / 1e9, "nvlink_peak_GBps": 770.0,
                     "frac_of_nvlink_peak": rho * gbytes / (kernel_ms * 1e-3) / 1e9 / 770.0}}))
