"""GPU: the two-layer max-pool aggregator (TwoMaxLayerPoolingAggregator, aggregator_type="twomaxpool").

* K5 (gs_maxpool2_mlp_fused) against the operand-exact contract of oracle/pool2_forward.py: grid inputs bit for bit
  (NaN in every pad column and every row no group reads, ids outside the table, one group reading one id k times), the
  unfused bf16 chain bit for bit on the same grid inputs, random operands within the derived bound (the largest ratios
  are printed at the end), and the launches outside the limits.
* The model: forward against a float64 torch reference in fp32, tf32x3 and bf16; graphed(B) replays equal eager calls.
* The model: in bf16 the forward launches K5 once per hop.
* Training: supervised loss and gradients against torch-CPU autograd (dropout 0 and 0.5 with the oracle's masks,
  identity_dim 0 and 16), the unsupervised three-pass loss and gradients against torch-CPU autograd (identity_dim 8),
  five clipped-Adam steps against a CPU twin, graphed_train_step replays equal to an eager twin (supervised, and the
  unsupervised step at dropout 0.5), two runs bit-identical, a peak-memory bound, a few steps on toy-ppi,
  full-neighbourhood inference against oracle.full_neighbor's layer with two Dense layers, and the refusals.

tests/test_pool2_forward_numerics_cpu.py shows on a numpy emulation that the K5 checks reject subtly wrong kernels."""
import numpy as np
import pytest
import torch

from conftest import load_golden, rel_err
from oracle import dropout as od
from oracle import pool2_forward as p2
from oracle import torch_ref

pytestmark = pytest.mark.gpu

SIZES = {"small": (512, 256), "big": (1024, 512)}
BAD_IDS = (-1, -7, -2 ** 31, 2 ** 31 - 1)             # plus n_rows and n_rows + 5: all read the last row
# (name, n_groups or "G-1" / "G+1" / "odd" in terms of G = 128 // k, k, K, size, "ids" | "row0")
CASES = [
    ("k1_K1", 1, 1, 1, "small", "ids"),
    ("k2_K5", "G-1", 2, 5, "big", "row0"),
    ("k25_K64", "G+1", 25, 64, "small", "ids"),
    ("k25_K602_big", "odd", 25, 602, "big", "ids"),
    ("k128_K640", 3, 128, 640, "small", "ids"),
    ("k128_K602", "odd", 128, 602, "big", "row0"),
    ("bench", 5120, 25, 602, "small", "ids"),              # configs[2]'s hop-2 launch of layer 0
]
MEASURED = {}


@pytest.fixture(scope="module")
def gs():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    import graphsage_b200
    graphsage_b200._lib.lib()
    yield graphsage_b200
    graphsage_b200.set_default_math("fp32")
    if MEASURED:
        print("\nK5 forward, measured on %s:" % torch.cuda.get_device_name())
        for name, (worst, rms) in sorted(MEASURED.items()):
            print("  %-14s worst |err| / bound = %.3e   rms = %.3e" % (name, worst, rms))


def case_inputs(case, grid, seed=0):
    name, spec, k, K, size, form = case
    h1, h2 = SIZES[size]
    G = 128 // k
    n = {"G-1": max(G - 1, 1), "G+1": G + 1, "odd": 7 * G + 3}.get(spec, spec)
    rs = np.random.RandomState(seed + 1000 * k + 7 * K + h1)
    pitch = (K + 7) // 8 * 8 + 8
    if form == "ids":
        n_rows = 2048
        pool = rs.choice(np.arange(1, n_rows - 1), size=200, replace=False)   # row 0 stays NaN
        ids = pool[rs.randint(0, pool.size, size=n * k)].astype(np.int64)
        ids[:k] = pool[0]
        bad = np.array(BAD_IDS + (n_rows, n_rows + 5), dtype=np.int64)
        pos = np.arange(k, min(n * k, k + bad.size))
        ids[pos] = bad[np.arange(pos.size) % bad.size]
        ids, row0, live = ids.astype(np.int32), 0, np.concatenate([pool, [n_rows - 1]])
    else:
        n_rows = max(600, n * k // 2 + 10)
        row0 = n_rows - max(1, n * k // 2)                  # runs past the table: the tail reads the last row
        ids, live = None, np.arange(row0, n_rows)
    table = np.full((n_rows, pitch), np.nan, np.float32)
    if grid:       # X on 2^-2, W on 2^-4, biases on 2^-6: both layers' fp32 sums exact (p2.grid_reference asserts it)
        vals = rs.randint(-4, 5, size=(live.size, K)) / 4.0
        W1, W2 = rs.randint(-4, 5, size=(K, h1)) / 16.0, rs.randint(-4, 5, size=(h1, h2)) / 16.0
        b1, b2 = rs.randint(-16, 17, size=h1) / 64.0, rs.randint(-16, 17, size=h2) / 64.0
    else:
        vals = p2.pf.nu.bf16_rne(rs.randn(live.size, K))
        W1, W2 = rs.randn(K, h1) / np.sqrt(K), rs.randn(h1, h2) / np.sqrt(h1 / 2)
        b1, b2 = rs.randn(h1) * 0.1, rs.randn(h2) * 0.1
    table[live, :K] = vals
    b2 = b2.astype(np.float32)
    b2[h2 - 1] = -4096.0                                    # every pre2 + b2 < 0: output 0
    return dict(table=table, n_rows=n_rows, K=K, k=k, n=n, h1=h1, h2=h2, ids=ids, row0=row0,
                W1=W1.astype(np.float32), b1=b1.astype(np.float32), W2=W2.astype(np.float32), b2=b2)


def _dev(gs, inp):
    t = lambda a: None if a is None else torch.from_numpy(a).cuda()   # noqa: E731
    return dict(table=t(inp["table"]).to(torch.bfloat16), ids=t(inp["ids"]), W1=t(inp["W1"]), b1=t(inp["b1"]),
                W2=t(inp["W2"]), b2=t(inp["b2"]), p1=gs.ops.PackedMlpWeights(), p2=gs.ops.PackedMlpWeights())


def _k5(gs, inp, d, out=None):
    return gs.ops.maxpool2_mlp_fused(d["table"][:, :inp["K"]], inp["n"], inp["k"], d["W1"], d["b1"], d["p1"], d["W2"],
                                     d["b2"], d["p2"], row_ids=d["ids"], row0=inp["row0"], out=out)


def _X(inp):
    idx = torch.from_numpy(p2.row_index(inp["n_rows"], inp["n"], inp["k"], inp["ids"], inp["row0"])).cuda()
    return torch.from_numpy(inp["table"][:, :inp["K"]]).cuda()[idx]


def _run(gs, inp, d):
    """K5 into a column slice of a NaN-filled buffer (left NaN around it), and again: the same bits."""
    n, h2 = inp["n"], inp["h2"]
    full = torch.full((n + 2, h2 + 9), float("nan"), device="cuda")
    out = _k5(gs, inp, d, out=full[:n, 5:5 + h2])
    again = _k5(gs, inp, d)
    torch.cuda.synchronize()
    rest = torch.cat([full[n:].reshape(-1), full[:n, :5].reshape(-1), full[:n, 5 + h2:].reshape(-1)])
    assert bool(torch.isnan(rest).all()), "wrote outside the output slice"
    assert torch.equal(out.view(torch.int32), again.view(torch.int32)), "two calls differ"
    return out


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_k5_grid_inputs_bit_for_bit(gs, case):
    inp = case_inputs(case, grid=True)
    ref = p2.grid_reference(_X(inp), inp["W1"], inp["b1"], inp["W2"], inp["b2"], inp["k"])
    assert bool((ref[:, -1] == 0).all()) and bool((ref > 0).any())
    out = _run(gs, inp, _dev(gs, inp))
    if not p2.same_values(out, ref):
        bad = torch.nonzero((out + 0.0).view(torch.int32) != (ref + 0.0).view(torch.int32))
        pytest.fail("%s: %d elements differ, first %s: got %r want %r" % (case[0], bad.shape[0], bad[0].tolist(),
                                                                         float(out[tuple(bad[0])]), float(ref[tuple(bad[0])])))


@pytest.mark.parametrize("case", [CASES[2], CASES[3], CASES[6]], ids=["k25_K64", "k25_K602_big", "bench"])
def test_k5_equals_the_unfused_bf16_chain_on_grid_inputs(gs, case):
    """gs_gather_rows_f32 -> Dense (bf16 GEMM, bias + ReLU) -> Dense -> gs_segment_max: the same operands, so the same
    bits on grid inputs."""
    inp = case_inputs(case, grid=True)
    d = _dev(gs, inp)
    agg = gs.TwoMaxLayerPoolingAggregator(inp["K"], 8, model_size=case[4])
    for layer, W, b in zip(agg.mlp_layers, (d["W1"], d["W2"]), (d["b1"], d["b2"])):
        layer.vars["weights"], layer.vars["bias"] = W, b
    agg.math = gs.ops.MATH_BF16
    ids = d["ids"] if d["ids"] is not None else None
    n, k = inp["n"], inp["k"]
    rows = gs.ops.gather_rows_f32(d["table"][:, :inp["K"]], ids=None if ids is None else ids[:n * k], row0=inp["row0"],
                                  n=n * k)
    chain = gs.ops.segment_max(agg._mlp(rows), n, k)
    assert p2.same_values(chain, _run(gs, inp, d))


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_k5_random_operands_within_the_derived_bound(gs, case):
    inp = case_inputs(case, grid=False)
    refs = p2.bounded_reference(_X(inp), inp["W1"], inp["b1"], inp["W2"], inp["b2"], inp["k"])
    ok, worst, rms = p2.check_bounded(_run(gs, inp, _dev(gs, inp)), *refs)
    MEASURED[case[0]] = (worst, rms)
    assert ok, (case[0], worst, rms)


def test_k5_refusals_and_the_aggregator_falls_back(gs):
    table = torch.zeros((64, 648), dtype=torch.bfloat16, device="cuda")
    ids = torch.zeros(129 * 4, dtype=torch.int32, device="cuda")
    W1, W2 = torch.zeros((64, 512), device="cuda"), torch.zeros((512, 256), device="cuda")
    P = gs.ops.PackedMlpWeights
    with pytest.raises(RuntimeError, match="k <= 128"):
        gs.ops.maxpool2_mlp_fused(table[:, :64], 2, 129, W1, None, P(), W2, None, P(), row_ids=ids)
    with pytest.raises(RuntimeError, match="K <= 640"):
        gs.ops.maxpool2_mlp_fused(table[:, :641], 2, 3, torch.zeros((641, 512), device="cuda"), None, P(), W2, None, P(),
                                  row_ids=ids)
    with pytest.raises(RuntimeError, match="h2 % 256 == 0"):
        gs.ops.maxpool2_mlp_fused(table[:, :64], 2, 3, W1, None, P(), torch.zeros((512, 384), device="cuda"), None, P(),
                                  row_ids=ids)
    with pytest.raises(RuntimeError, match="h1 % 128 == 0"):
        gs.ops.maxpool2_mlp_fused(table[:, :64], 2, 3, torch.zeros((64, 320), device="cuda"), None, P(),
                                  torch.zeros((320, 256), device="cuda"), None, P(), row_ids=ids)
    # K must name W1's rows (the packed images hold ceil(rows / 64) K-blocks): a mismatch is refused, in K4's wrapper too
    for K in (65, 0):
        with pytest.raises(ValueError, match="does not match"):
            gs.ops.maxpool2_mlp_fused(table[:, :64], 2, 3, W1, None, P(), W2, None, P(), row_ids=ids, K=K)
        with pytest.raises(ValueError, match="does not match"):
            gs.ops.maxpool_mlp_fused(table[:, :64], 2, 3, W1, None, P(), row_ids=ids, K=K)
    with pytest.raises(ValueError, match="does not match"):
        gs.ops.maxpool2_mlp_fused(table[:, :200], 2, 3, torch.zeros((130, 512), device="cuda"), None, P(), W2, None, P(),
                                  row_ids=ids, K=64)
    # a fanout above 128 in bf16: the aggregator takes the materialised chain, bit for bit
    rs = np.random.RandomState(4)
    feats = torch.from_numpy(p2.pf.nu.bf16_rne(rs.randn(300, 40))).cuda()
    agg = gs.TwoMaxLayerPoolingAggregator(40, 16)
    agg.math = gs.ops.MATH_BF16
    for layer in agg.mlp_layers:
        layer.vars["bias"].normal_()
    s = gs.ops.Seg(3, 130, self_ids=torch.arange(3, dtype=torch.int32, device="cuda"),
                   neigh_ids=torch.from_numpy(rs.randint(0, 300, 390).astype(np.int32)).cuda())
    assert not agg._fused_ok(feats, [s])
    got = agg.aggregate_rows(feats, [s])
    want = agg._finish(agg._pooled_parts(feats, [s]), agg._combine())
    assert torch.equal(got, want)


# ---------------------------------------------------------------- the model
def _cpu_outputs(adj, feats, seeds, fan, aggs, concat, seed, counter, drop=None, normalize=True):
    """float64-capable torch reference of the sampled forward (models.py:254-330 with aggregators.py:330-361); drop:
    (seed, first call, rate) - the MLP inputs of both Dense layers per (layer, hop) masked in the plan's order."""
    adj_t, feats_t, seeds_t = torch.from_numpy(adj), feats, torch.from_numpy(seeds)
    L = len(fan)
    samples, sup = [seeds_t], 1
    for k in range(L):
        sup *= fan[L - k - 1]
        samples.append(torch_ref.sample_padded(adj_t, samples[k], fan[L - k - 1], seed, counter + k).reshape(-1))
    hidden = [feats_t.index_select(0, s.long()) for s in samples]
    call = None if drop is None else drop[1]

    def dr(x):
        nonlocal call
        if drop is None:
            return x
        m = torch.from_numpy(od.keep_mask(drop[0], call, drop[2], np.arange(x.shape[0]), x.shape[1]))
        call += 1
        return torch.where(m, x / od.keep_prob(drop[2]), torch.zeros_like(x))

    for layer in range(L):
        a, last, nxt = aggs[layer], layer == L - 1, []
        for hop in range(L - layer):
            k = fan[L - hop - 1]
            neigh, selfv = hidden[hop + 1], hidden[hop]
            n = selfv.shape[0]
            h = torch.relu(dr(neigh) @ a["W1"] + a["b1"])
            h = torch.relu(dr(h) @ a["W2"] + a["b2"]).reshape(n, k, -1).amax(dim=1)
            fs, fn = selfv @ a["self_weights"], h @ a["neigh_weights"]
            y = torch.cat([fs, fn], dim=1) if concat else fs + fn
            if "bias" in a:
                y = y + a["bias"]
            nxt.append(y if last else torch.relu(y))
        hidden = nxt
    out = hidden[0]
    if normalize:
        out = out / torch.sqrt(torch.clamp((out * out).sum(dim=1, keepdim=True), min=1e-12))
    return out


def _weights(m, dtype=torch.float32, grad=False):
    aggs = []
    for a in m.aggregators:
        d = {k: v.detach().cpu() for k, v in a.vars.items()}
        for i, layer in enumerate(a.mlp_layers):
            d["W%d" % (i + 1)], d["b%d" % (i + 1)] = layer.vars["weights"].detach().cpu(), layer.vars["bias"].detach().cpu()
        aggs.append({k: v.to(dtype).clone().requires_grad_(grad) for k, v in d.items()})
    return aggs


def _nonzero_biases(m, seed=2):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    for a in m.aggregators:
        for layer in a.mlp_layers:
            b = layer.vars["bias"]
            b.data.add_(torch.randn(b.shape, generator=gen, device=b.device) * 0.1)


@pytest.mark.parametrize("math,tol", [("fp32", 1e-4), ("tf32x3", 1e-4), ("bf16", 2e-2)])
def test_model_forward_against_the_reference_and_graphed_replays(gs, math, tol):
    g = load_golden("khop")
    adj, feats = g["adj"], g["feats"]
    rs = np.random.RandomState(3)
    B = 32
    gs.set_default_math(math)
    try:
        sampler = gs.UniformNeighborSampler(torch.from_numpy(adj).cuda(), seed=123)
        infos = [gs.SAGEInfo("node", sampler, 10, 64), gs.SAGEInfo("node", sampler, 5, 64)]
        m = gs.SampleAndAggregate({"batch_size": B, "dropout": 0.}, torch.from_numpy(feats).cuda(),
                                  torch.from_numpy(adj).cuda(), None, infos, concat=True, aggregator_type="twomaxpool")
        seeds = rs.randint(0, adj.shape[0] - 1, size=B).astype(np.int32)
        out = m.forward(torch.from_numpy(seeds))
        _nonzero_biases(m)
        ref = _cpu_outputs(adj, torch.from_numpy(feats).double(), seeds, [10, 5], _weights(m, torch.float64), True, 123, 0)
        assert tuple(out.shape) == (B, 128)
        sampler.counter = 0
        out = m.forward(torch.from_numpy(seeds))
        assert rel_err(out.cpu().numpy(), ref.numpy()) < tol
        if math == "bf16":                            # K5 ran: one launch per hop (layer 0: two hops, layer 1: one)
            gs.ops.PROBE = {}
            try:
                m.forward(torch.from_numpy(seeds))
                torch.cuda.synchronize()
                launches = sum(len(v) for name, v in gs.ops.PROBE.items() if name.startswith("maxpool2_mlp/"))
            finally:
                gs.ops.PROBE = None
            assert launches == 3
        # graphed(B): replays equal eager calls from the same sampler state
        c = sampler.counter
        batches = [torch.from_numpy(rs.randint(0, adj.shape[0] - 1, size=B).astype(np.int32)).cuda() for _ in range(3)]
        eager = [m.forward(ids).clone() for ids in batches]
        sampler.counter = c
        run = m.graphed(B)
        for i, (ids, want) in enumerate(zip(batches, eager)):
            assert torch.equal(run(ids), want), i
        run.close()
    finally:
        gs.set_default_math("fp32")


def _supervised(gs, concat=True, d=0, rate=0.0, math="fp32", fan=(4, 3), dim=16, C=5):
    g = load_golden("khop")
    gs.inits.manual_seed(11)
    gs.set_default_math(math)
    try:
        sampler = gs.UniformNeighborSampler(torch.from_numpy(g["adj"]).cuda(), seed=123)
        sampler.counter = 40
        infos = [gs.SAGEInfo("node", sampler, fan[0], dim), gs.SAGEInfo("node", sampler, fan[1], dim)]
        m = gs.SupervisedGraphsage(C, {"batch_size": 16, "dropout": rate}, torch.from_numpy(g["feats"]).cuda(),
                                   torch.from_numpy(g["adj"]).cuda(), None, infos, concat=concat,
                                   aggregator_type="twomaxpool", sigmoid_loss=True, learning_rate=0.01, weight_decay=1e-3,
                                   identity_dim=d, dropout_seed=99)
    finally:
        gs.set_default_math("fp32")
    _nonzero_biases(m)
    return m, g


def _cpu_loss(m, g, seeds, labels, rate, concat):
    aggs = _weights(m, grad=True)
    head = {k: v.detach().cpu().clone().requires_grad_(True) for k, v in m.node_pred_vars.items()}
    feats = torch.from_numpy(g["feats"])
    emb = None
    if getattr(m, "embeds", None) is not None:
        emb = m.embeds.detach().cpu().clone().requires_grad_(True)
        feats = torch.cat([emb, feats], dim=1)                  # the [N+1, d + F] table: embeddings first
    drop = (99, 0, rate) if rate else None
    out = _cpu_outputs(g["adj"], feats, seeds, [4, 3], aggs, concat, 123, 40, drop=drop)
    if rate:
        out = torch.where(torch.from_numpy(od.keep_mask(99, 6, rate, np.arange(out.shape[0]), out.shape[1])),
                          out / od.keep_prob(rate), torch.zeros_like(out))
    logits = out @ head["weights"] + head["bias"]
    ref = torch.nn.functional.binary_cross_entropy_with_logits(logits, torch.from_numpy(labels))
    for a in aggs:                                    # the reference decays aggregator.vars only, not the Dense variables
        for k in ("neigh_weights", "self_weights"):
            ref = ref + 1e-3 * 0.5 * (a[k] * a[k]).sum()
    for v in head.values():
        ref = ref + 1e-3 * 0.5 * (v * v).sum()
    ref.backward()
    return ref, aggs, head, emb


@pytest.mark.parametrize("concat,d,rate", [(True, 0, 0.0), (False, 0, 0.0), (True, 16, 0.0), (True, 0, 0.5),
                                           (False, 16, 0.5)])
def test_supervised_loss_and_gradients_match_cpu_autograd(gs, concat, d, rate):
    m, g = _supervised(gs, concat, d, rate)
    rs = np.random.RandomState(5)
    seeds = rs.randint(0, g["adj"].shape[0] - 1, size=16).astype(np.int32)
    labels = (rs.rand(16, 5) < 0.3).astype(np.float32)
    ref, aggs, head, emb = _cpu_loss(m, g, seeds, labels, rate, concat)
    loss = m.loss(torch.from_numpy(seeds), torch.from_numpy(labels), dropout=rate)
    loss.backward()
    assert abs(float(loss) - float(ref)) < 1e-5 * max(1.0, abs(float(ref)))
    for a, ra in zip(m.aggregators, aggs):
        got = {k: v.grad for k, v in a.vars.items()}
        for i, layer in enumerate(a.mlp_layers):
            got["W%d" % (i + 1)], got["b%d" % (i + 1)] = layer.vars["weights"].grad, layer.vars["bias"].grad
        for k, v in got.items():                       # a bias compares as one row (rel_err is per row)
            assert rel_err(v.cpu().numpy().reshape(-1, v.shape[-1]), ra[k].grad.numpy().reshape(-1, v.shape[-1]),
                           floor=1e-8) < 2e-4, k
    if emb is not None:
        assert rel_err(m.embeds.grad.cpu().numpy(), emb.grad.numpy(), floor=1e-8) < 2e-4
    assert m.dropout_counter == (7 if rate else 0)


def test_five_adam_steps_track_a_cpu_run_and_two_runs_are_bit_identical(gs):
    runs = []
    for _ in range(2):
        m, g = _supervised(gs)
        rs = np.random.RandomState(6)
        losses = []
        torch.cuda.synchronize()
        before = torch.cuda.memory_allocated()           # other tests' tensors may still be alive
        torch.cuda.reset_peak_memory_stats()
        for _ in range(5):
            seeds = rs.randint(0, g["adj"].shape[0] - 1, size=16).astype(np.int32)
            labels = (rs.rand(16, 5) < 0.3).astype(np.float32)
            losses.append(m.train_step(torch.from_numpy(seeds), torch.from_numpy(labels)))
        torch.cuda.synchronize()
        assert torch.cuda.max_memory_allocated() - before < 256 * 2 ** 20   # peak above what the steps found
        runs.append((torch.stack(losses), [p.detach().clone() for p in m.parameters()]))
    assert torch.equal(runs[0][0], runs[1][0]) and all(torch.equal(p, q) for p, q in zip(runs[0][1], runs[1][1]))
    # the CPU twin: the same five steps as torch-CPU autograd + torch.optim.Adam with clipping
    m, g = _supervised(gs)
    aggs = _weights(m, grad=True)
    head = {k: v.detach().cpu().clone().requires_grad_(True) for k, v in m.node_pred_vars.items()}
    params = [t for a in aggs for t in a.values()] + list(head.values())
    opt = torch.optim.Adam(params, lr=0.01)
    rs = np.random.RandomState(6)
    for step in range(5):
        seeds = rs.randint(0, g["adj"].shape[0] - 1, size=16).astype(np.int32)
        labels = (rs.rand(16, 5) < 0.3).astype(np.float32)
        out = _cpu_outputs(g["adj"], torch.from_numpy(g["feats"]), seeds, [4, 3], aggs, True, 123, 40 + 2 * step)
        ref = torch.nn.functional.binary_cross_entropy_with_logits(out @ head["weights"] + head["bias"],
                                                                   torch.from_numpy(labels))
        for a in aggs:
            for k in ("neigh_weights", "self_weights"):
                ref = ref + 1e-3 * 0.5 * (a[k] * a[k]).sum()
        for v in head.values():
            ref = ref + 1e-3 * 0.5 * (v * v).sum()
        opt.zero_grad()
        ref.backward()
        for p in params:
            p.grad.clamp_(-5.0, 5.0)
        opt.step()
        assert abs(float(runs[0][0][step]) - float(ref)) < 1e-4 * max(1.0, abs(float(ref))), step
    # m.parameters()'s order: every aggregator's vars, then every Dense's weights and bias, then the head
    cpu = [ra[k] for a, ra in zip(m.aggregators, aggs) for k in a.vars]
    cpu += [ra[k] for ra in aggs for k in ("W1", "b1", "W2", "b2")] + [head["weights"], head["bias"]]
    # Adam's step m / sqrt(v) is scale-free: an element whose gradient is near 0 moves by up to lr on rounding noise
    for p, q in zip(runs[0][1], cpu):
        assert tuple(p.shape) == tuple(q.shape)
        assert rel_err(p.reshape(1, -1).cpu().numpy(), q.detach().reshape(1, -1).numpy()) < 2e-3


def test_unsupervised_loss_and_gradients_match_cpu_autograd(gs):
    """The unsupervised three-pass loss (batch1, batch2, unigram negatives through the same aggregators; models.py:332-405)
    with identity_dim 8, against torch-CPU autograd on the same samples and negatives."""
    import oracle
    g = load_golden("khop")
    rs = np.random.RandomState(11)
    adj, feats = g["adj"], g["feats"]
    n, B, NEG, d = adj.shape[0] - 1, 16, 20, 8
    deg = rs.randint(1, 40, size=n).astype(np.float64)
    b1 = rs.randint(0, n, size=B).astype(np.int32)
    b2 = rs.randint(0, n, size=B).astype(np.int32)
    fan = [4, 3]
    gs.set_default_math("fp32")
    gs.inits.manual_seed(11)
    sampler = gs.UniformNeighborSampler(torch.from_numpy(adj).cuda(), seed=123)
    infos = [gs.SAGEInfo("node", sampler, fan[0], 12), gs.SAGEInfo("node", sampler, fan[1], 12)]
    m = gs.UnsupervisedGraphsage({"batch_size": B, "dropout": 0.}, torch.from_numpy(feats).cuda(),
                                 torch.from_numpy(adj).cuda(), deg, infos, concat=True, aggregator_type="twomaxpool",
                                 neg_sample_size=NEG, learning_rate=0.01, weight_decay=1e-3, seed=77, identity_dim=d)
    _nonzero_biases(m)
    aggs = _weights(m, grad=True)
    E = m.embeds.detach().cpu().clone().requires_grad_(True)
    table = torch.cat([E, torch.from_numpy(feats)], dim=1)
    neg = oracle.sample_unigram(deg, NEG, 77, 0)
    o1 = _cpu_outputs(adj, table, b1, fan, aggs, True, 123, 0)
    o2 = _cpu_outputs(adj, table, b2, fan, aggs, True, 123, 2)
    on = _cpu_outputs(adj, table, np.asarray(neg).astype(np.int32), fan, aggs, True, 123, 4)
    ref = torch.nn.functional.softplus(-(o1 * o2).sum(1)).sum() + torch.nn.functional.softplus(o1 @ on.t()).sum()
    for a in aggs:                                    # the reference decays aggregator.vars only, not the Dense variables
        for k in ("neigh_weights", "self_weights"):
            ref = ref + 1e-3 * 0.5 * (a[k] * a[k]).sum()
    ref = ref / B
    ref.backward()
    loss = m.loss(torch.from_numpy(b1), torch.from_numpy(b2))
    loss.backward()
    assert abs(float(loss.detach()) - float(ref.detach())) < 1e-5 * max(1.0, abs(float(ref.detach())))
    for a, ra in zip(m.aggregators, aggs):
        got = {k: v.grad for k, v in a.vars.items()}
        for i, layer in enumerate(a.mlp_layers):
            got["W%d" % (i + 1)], got["b%d" % (i + 1)] = layer.vars["weights"].grad, layer.vars["bias"].grad
        for k, v in got.items():
            assert rel_err(v.cpu().numpy().reshape(-1, v.shape[-1]), ra[k].grad.numpy().reshape(-1, v.shape[-1]),
                           floor=1e-8) < 2e-4, k
    assert rel_err(m.embeds.grad.cpu().numpy(), E.grad.numpy(), floor=1e-8) < 2e-4


def test_unsupervised_graphed_replays_equal_an_eager_twin(gs):
    g = load_golden("khop")
    rs = np.random.RandomState(7)

    def build():
        gs.inits.manual_seed(11)
        sampler = gs.UniformNeighborSampler(torch.from_numpy(g["adj"]).cuda(), seed=7)
        infos = [gs.SAGEInfo("node", sampler, 4, 16), gs.SAGEInfo("node", sampler, 3, 16)]
        m = gs.UnsupervisedGraphsage({"batch_size": 16, "dropout": 0.5}, torch.from_numpy(g["feats"]).cuda(),
                                     torch.from_numpy(g["adj"]).cuda(), torch.from_numpy(np.ones(g["adj"].shape[0] - 1)),
                                     infos, aggregator_type="twomaxpool", neg_sample_size=5, learning_rate=0.01,
                                     identity_dim=8, dropout_seed=99)
        return m

    m, twin = build(), build()
    gs.make_adam_capturable(twin.optimizer)
    n = g["adj"].shape[0] - 1
    batches = [(torch.from_numpy(rs.randint(0, n, 16).astype(np.int32)), torch.from_numpy(rs.randint(0, n, 16).astype(np.int32)))
               for _ in range(3)]
    step = m.graphed_train_step(16)
    for b1, b2 in batches:
        assert torch.equal(step(b1.cuda(), b2.cuda()), twin.train_step(b1, b2))
    assert all(torch.equal(p, q) for p, q in zip(m.parameters(), twin.parameters()))


def test_supervised_graphed_train_step_equals_an_eager_twin(gs):
    m, _ = _supervised(gs, rate=0.5, d=16, math="tf32x3")
    twin, g = _supervised(gs, rate=0.5, d=16, math="tf32x3")
    gs.make_adam_capturable(twin.optimizer)
    step = m.graphed_train_step(16)
    rs = np.random.RandomState(9)
    for _ in range(4):
        ids = torch.from_numpy(rs.randint(0, g["adj"].shape[0] - 1, size=16).astype(np.int32))
        labels = torch.from_numpy((rs.rand(16, 5) < 0.3).astype(np.float32))
        assert torch.equal(step(ids.cuda(), labels.cuda()), twin.train_step(ids, labels))
    assert all(torch.equal(p, q) for p, q in zip(m.parameters(), twin.parameters()))
    assert m.dropout_counter == twin.dropout_counter > 0


def test_full_neighbor_inference_and_the_refusals(gs):
    m, g = _supervised(gs, concat=True)
    adj = g["adj"]
    n = adj.shape[0] - 1
    rs = np.random.RandomState(1)
    deg = rs.randint(0, 6, size=n)
    indptr = np.concatenate([[0], np.cumsum(deg)]).astype(np.int64)
    indices = rs.randint(0, n, size=int(indptr[-1])).astype(np.int32)
    ids = np.arange(0, n, 7, dtype=np.int32)
    csr = (torch.from_numpy(indptr).cuda(), torch.from_numpy(indices).cuda(), torch.from_numpy(ids).cuda())
    out = m.full_neighbor_embeddings(*csr)
    ws = [{k: v.numpy() for k, v in w.items()} for w in _weights(m)]
    ref = p2.full_neighbor_embeddings(g["feats"], indptr, indices, ws, True, node_ids=ids)
    assert rel_err(out.cpu().numpy(), ref) < 1e-4
    with pytest.raises(NotImplementedError, match="twomaxpool"):
        m.full_neighbor_train_step(*csr, torch.zeros((ids.size, 5)))
    with pytest.raises(NotImplementedError, match="twomaxpool"):
        m.full_neighbor_minibatch_loss(*csr, torch.zeros((ids.size, 5)))
    with pytest.raises(NotImplementedError, match="one MLP layer"):
        gs.SupervisedGraphsage(5, {"batch_size": 16, "dropout": 0.}, torch.from_numpy(g["feats"]).cuda(),
                               torch.from_numpy(adj).cuda(), None, m.layer_infos, aggregator_type="twomaxpool",
                               fused_pool=True)


def test_a_few_steps_on_toy_ppi(gs):
    """Twenty supervised steps of the class on a slice of the reference's toy-ppi (bf16 math, so K5 in the forward):
    the loss falls, evaluation over whole neighbourhoods runs and is repeatable."""
    from test_walks_cpu import toy_graph
    from graphsage_b200.minibatch import NodeMinibatchIterator
    g = load_golden("toy_ppi")
    G = toy_graph()
    id2idx = {u: i for i, u in enumerate(G.nodes())}
    labels = (np.asarray(g["labels"]) > 0).astype(np.float32)
    it = NodeMinibatchIterator(G, id2idx, None, {u: labels[i] for i, u in enumerate(G.nodes())}, labels.shape[1],
                               batch_size=64, max_degree=25, rng=np.random.RandomState(0))
    n = len(id2idx)
    feats = torch.zeros((n + 1, 50), device="cuda")
    feats[:n] = torch.from_numpy(np.asarray(g["feats"], np.float32)).cuda()
    gs.inits.manual_seed(3)
    adj = torch.from_numpy(it.adj).cuda()
    sampler = gs.UniformNeighborSampler(adj, seed=1)
    infos = [gs.SAGEInfo("node", sampler, 10, 64), gs.SAGEInfo("node", sampler, 5, 64)]
    gs.set_default_math("bf16")
    try:
        m = gs.SupervisedGraphsage(labels.shape[1], {"batch_size": 64, "dropout": 0.}, feats, adj, None, infos,
                                   aggregator_type="twomaxpool", sigmoid_loss=True, learning_rate=0.01)
    finally:
        gs.set_default_math("fp32")
    train = np.array([id2idx[u] for u in G.nodes() if not G.node[u]["val"] and not G.node[u]["test"]])
    rs = np.random.RandomState(0)
    eval_ids = rs.choice(train, 256).astype(np.int32)
    before = float(m.loss(torch.from_numpy(eval_ids), torch.from_numpy(labels[eval_ids])))
    for _ in range(20):
        ids = rs.choice(train, 64).astype(np.int32)
        m.train_step(torch.from_numpy(ids), torch.from_numpy(labels[ids]))
    after = float(m.loss(torch.from_numpy(eval_ids), torch.from_numpy(labels[eval_ids])))
    assert np.isfinite(after) and after < before, (before, after)
    val = np.array([id2idx[u] for u in G.nodes() if G.node[u]["val"]], dtype=np.int32)
    indptr, indices = it.neighbor_csr(test=True)
    preds = m.full_neighbor_predict(indptr, indices, val)
    assert preds.shape == (len(val), labels.shape[1]) and torch.equal(preds, m.full_neighbor_predict(indptr, indices, val))
