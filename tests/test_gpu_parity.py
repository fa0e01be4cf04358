"""GPU: parity of the CUDA path (through the C-ABI) against the oracle and the committed golden
vectors.  Bit-exact for integer work; fp32 layer outputs within 1e-4 relative (north_star)."""
import numpy as np
import pytest
import torch

import oracle
from conftest import bf16_round, elem_err, load_golden, rel_err

pytestmark = pytest.mark.gpu

TOL = 1e-4   # north_star: "fp32 layer outputs within 1e-4 rel"


@pytest.fixture(scope="module")
def gs():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    import graphsage_b200
    graphsage_b200._lib.lib()        # raises if the .so is missing: no silent fallback
    return graphsage_b200


def dev(x, dtype=None):
    t = torch.as_tensor(np.ascontiguousarray(x))
    if dtype is not None:
        t = t.to(dtype)
    return t.cuda()


MATHS = ["fp32", "tf32x3"]


# ---------------------------------------------------------------- K1 sampler
def test_sampler_golden_bit_exact(gs):
    g = load_golden("sampler")
    for ci in range(int(g["n_cases"])):
        out = gs.ops.sample_padded(dev(g["adj%d" % ci]), dev(g["ids%d" % ci]), int(g["k%d" % ci]),
                                   int(g["seed%d" % ci]), int(g["counter%d" % ci]))
        assert out.dtype == torch.int32
        np.testing.assert_array_equal(out.cpu().numpy(), g["out%d" % ci])


def test_sampler_class_counter_and_swap(gs):
    rs = np.random.RandomState(3)
    n, md = 1000, 128
    adj = rs.randint(0, n, size=(n + 1, md)).astype(np.int32)
    adj[n] = n
    ids = rs.randint(0, n + 1, size=777).astype(np.int32)
    s = gs.UniformNeighborSampler(dev(adj), seed=11)
    a = s((dev(ids), 10)).cpu().numpy()
    b = s((dev(ids), 25)).cpu().numpy()          # second call -> counter 1 -> fresh permutation
    np.testing.assert_array_equal(a, oracle.sample_padded(adj, ids, 10, 11, 0))
    np.testing.assert_array_equal(b, oracle.sample_padded(adj, ids, 25, 11, 1))
    # same column set for every row of a call (neigh_samplers.py:27), columns distinct
    pi = oracle.perm_prefix(11, 1, md, 25)
    assert len(set(pi.tolist())) == 25
    adj2 = np.roll(adj, 1, axis=1).copy()
    s.set_adj(dev(adj2))
    c = s((dev(ids), 25)).cpu().numpy()
    np.testing.assert_array_equal(c, oracle.sample_padded(adj2, ids, 25, 11, 2))
    # full-width sample, explicit permutation, device-side counter, empty batch
    full = gs.ops.sample_padded(dev(adj), dev(ids), md, 5, 9).cpu().numpy()
    np.testing.assert_array_equal(full, oracle.sample_padded(adj, ids, md, 5, 9))
    perm = rs.permutation(md).astype(np.int32)
    e = gs.ops.sample_padded(dev(adj), dev(ids), 7, 0, 0, col_perm=dev(perm)).cpu().numpy()
    np.testing.assert_array_equal(e, adj[ids][:, perm[:7]])
    cdev = torch.tensor([1 << 35], dtype=torch.int64).cuda()
    f = gs.ops.sample_padded(dev(adj), dev(ids), 10, 11, 4, counter_dev=cdev).cpu().numpy()
    np.testing.assert_array_equal(f, oracle.sample_padded(adj, ids, 10, 11, 4 + (1 << 35)))
    assert gs.ops.sample_padded(dev(adj), dev(ids[:0]), 10, 1, 1).shape == (0, 10)
    with pytest.raises(RuntimeError, match="num_samples"):
        gs.ops.sample_padded(dev(adj), dev(ids), md + 1, 1, 1)
    oob = np.array([-5, n + 7], dtype=np.int32)             # out-of-range ids read the dummy row
    assert (gs.ops.sample_padded(dev(adj), dev(oob), 4, 1, 1).cpu().numpy() == n).all()


def test_sample_csr_bit_exact(gs):
    rs = np.random.RandomState(5)
    n = 5000
    deg = rs.randint(0, 60, size=n)
    deg[:4] = [0, 1, 25, 26]
    indptr = np.concatenate([[0], np.cumsum(deg)]).astype(np.int64)
    indices = rs.randint(0, n, size=int(indptr[-1])).astype(np.int32)
    ids = rs.randint(0, n, size=3333).astype(np.int32)
    ids[:4] = [0, 1, 2, 3]
    for k in (1, 10, 25, 32):
        for rep in (True, False):
            out = gs.ops.sample_csr(dev(indptr), dev(indices), dev(ids), k, 77, 5, rep, pad_id=n).cpu().numpy()
            np.testing.assert_array_equal(out, oracle.sample_csr(indptr, indices, ids, k, 77, 5, rep, pad_id=n))
    with pytest.raises(RuntimeError, match="not supported"):
        gs.ops.sample_csr(dev(indptr), dev(indices), dev(ids), 33, 1, 1)


# ---------------------------------------------------------------- K2 gather
@pytest.mark.parametrize("variant", [0, 1])
@pytest.mark.parametrize("F", [602, 50, 256, 7])
def test_gather_rows_exact(gs, variant, F):
    rs = np.random.RandomState(F)
    n = 4097
    feats = rs.randn(n + 1, F).astype(np.float32)
    ids = rs.randint(0, n + 1, size=10001).astype(np.int32)
    gs._lib.set_tuning("gather_variant", variant)
    try:
        P = gs.ops.pad_cols(F)
        table = torch.zeros((n + 1, P), dtype=torch.float32, device="cuda")
        table[:, :F] = dev(feats)
        out = gs.ops.gather_rows(table[:, :F], dev(ids))          # pitched table view (pitch 608 for F=602)
        np.testing.assert_array_equal(out.cpu().numpy(), feats[ids])
        out2 = gs.ops.gather_rows(dev(feats), dev(ids))           # dense pitch == F
        np.testing.assert_array_equal(out2.cpu().numpy(), feats[ids])
        outp = torch.empty((len(ids), P), dtype=torch.float32, device="cuda")
        gs.ops.gather_rows(table, dev(ids), out=outp)             # whole padded rows: the TMA bulk path
        np.testing.assert_array_equal(outp[:, :F].cpu().numpy(), feats[ids])
        bf = table.to(torch.bfloat16)
        ob = gs.ops.gather_rows(bf, dev(ids))
        assert torch.equal(ob, bf[dev(ids).long()])
    finally:
        gs._lib.set_tuning("gather_variant", 2)


@pytest.mark.parametrize("variant", [0, 1, 2])
def test_gather_mean_matches_numpy(gs, variant):
    rs = np.random.RandomState(9)
    n_src, F = 3000, 602
    P = gs.ops.pad_cols(F)
    feats = rs.randn(n_src, F).astype(np.float32)
    table = torch.full((n_src, P), 7.0, dtype=torch.float32, device="cuda")   # poison the pad columns
    table[:, :F] = dev(feats)
    src = table[:, :F]
    n0, k0, n1, k1 = 64, 10, 640, 25
    s0 = rs.randint(0, n_src, size=n0).astype(np.int32)
    s1 = rs.randint(0, n_src, size=n0 * k0).astype(np.int32)
    s2 = rs.randint(0, n_src, size=n1 * k1).astype(np.int32)
    gs._lib.set_tuning("gather_variant", variant)
    try:
        segs = [gs.ops.Seg(n0, k0, self_ids=dev(s0), neigh_ids=dev(s1), out_row0=0),
                gs.ops.Seg(n1, k1, self_ids=dev(s1), neigh_ids=dev(s2), out_row0=n0)]
        for include_self in (False, True):
            xs, xm = gs.ops.gather_mean(src, segs, include_self=include_self)
            xs, xm = xs.cpu().numpy(), xm.cpu().numpy()
            assert xs.shape == (n0 + n1, P) and (xs[:, F:] == 0).all() and (xm[:, F:] == 0).all()
            np.testing.assert_array_equal(xs[:, :F], feats[np.concatenate([s0, s1])])
            nb0 = feats[s1].reshape(n0, k0, F)
            nb1 = feats[s2].reshape(n1, k1, F)
            if include_self:
                ref = np.concatenate([(nb0.sum(1) + feats[s0]) / (k0 + 1), (nb1.sum(1) + feats[s1]) / (k1 + 1)])
            else:
                ref = np.concatenate([nb0.mean(1), nb1.mean(1)])
            assert rel_err(xm[:, :F], ref) < 1e-5
        # dense (id-free) form: rows addressed by ranges
        H = rs.randn(n0 + n0 * k0, 256).astype(np.float32)
        _, m = gs.ops.gather_mean(dev(H), [gs.ops.Seg(n0, k0, self_row0=0, neigh_row0=n0)], want_self=False)
        assert rel_err(m.cpu().numpy()[:, :256], H[n0:].reshape(n0, k0, 256).mean(1)) < 1e-5
    finally:
        gs._lib.set_tuning("gather_variant", 2)


@pytest.mark.parametrize("form", ["tma2", "tma", "ldg", "scalar", "bf16"])
def test_gather_mean_segments_of_any_size(gs, form):
    """A call's segments may come in any size order, empty ones included: each output row must use its own segment's
    fanout and ids (a row of a long segment followed by a shorter or empty one used to be placed in the later segment)."""
    rs = np.random.RandomState(17)
    n_src, F = 1000, 7 if form == "scalar" else 50
    feats = rs.randn(n_src, F).astype(np.float32)
    if form == "bf16":
        feats = bf16_round(feats)
    spec = [(40, 25), (0, 13), (9, 128), (17, 14)]
    segs, ref, row = [], [], 0
    for n, k in spec:
        s = rs.randint(0, n_src, size=n).astype(np.int32)
        nb = rs.randint(0, n_src, size=n * k).astype(np.int32)
        segs.append(gs.ops.Seg(n, k, self_ids=dev(s), neigh_ids=dev(nb), out_row0=row))
        ref.append(feats[nb].astype(np.float64).reshape(n, k, F).mean(1))
        row += n
    if form == "scalar":
        src = dev(feats)                                      # pitch 7: no 16-byte rows -> scalar kernel
    else:
        table = torch.zeros((n_src, gs.ops.pad_cols(F)), dtype=torch.float32, device="cuda")
        table[:, :F] = dev(feats)
        src = (table.to(torch.bfloat16) if form == "bf16" else table)[:, :F]
    gs._lib.set_tuning("gather_variant", {"tma2": 2, "tma": 1, "ldg": 0}.get(form, 2))
    try:
        _, xm = gs.ops.gather_mean(src, segs, want_self=False)
    finally:
        gs._lib.set_tuning("gather_variant", 2)
    assert rel_err(xm[:, :F].cpu().numpy(), np.vstack(ref)) < 1e-6


def test_gather_mean_odd_width_scalar_path(gs):
    rs = np.random.RandomState(2)
    x = rs.randn(500, 7).astype(np.float32)                  # pitch 7: no 16-B alignment -> scalar kernel
    ids = rs.randint(0, 500, size=30 * 4).astype(np.int32)
    sid = rs.randint(0, 500, size=30).astype(np.int32)
    xs, xm = gs.ops.gather_mean(dev(x), [gs.ops.Seg(30, 4, self_ids=dev(sid), neigh_ids=dev(ids))])
    np.testing.assert_array_equal(xs.cpu().numpy()[:, :7], x[sid])
    assert rel_err(xm.cpu().numpy()[:, :7], x[ids].reshape(30, 4, 7).mean(1)) < 1e-6


# ---------------------------------------------------------------- aggregators (golden = reference code under shim)
def _inject(agg, **weights):
    for k, v in weights.items():
        assert tuple(agg.vars[k].shape) == tuple(v.shape), (k, agg.vars[k].shape, v.shape)
        agg.vars[k] = dev(v)


@pytest.mark.parametrize("math", MATHS)
def test_aggregators_golden(gs, math):
    g = load_golden("aggregators")
    gs.set_default_math(math)
    s, n = dev(g["self"]), dev(g["neigh"])
    for c in (0, 1):
        agg = gs.MeanAggregator(50, 16, concat=bool(c))
        assert set(agg.vars) == {"neigh_weights", "self_weights"}
        _inject(agg, neigh_weights=g["mean_c%d_nw" % c], self_weights=g["mean_c%d_sw" % c])
        y = agg((s, n))
        assert tuple(y.shape) == (37, 16 * (1 + c))
        assert rel_err(y.cpu().numpy(), g["mean_c%d_out" % c]) < TOL
        agg = gs.MaxPoolingAggregator(50, 16, concat=bool(c))
        assert agg.hidden_dim == 512 and set(agg.mlp_layers[0].vars) == {"weights", "bias"}
        _inject(agg, neigh_weights=g["maxpool_c%d_nw" % c], self_weights=g["maxpool_c%d_sw" % c])
        _inject(agg.mlp_layers[0], weights=g["maxpool_c%d_mw" % c], bias=g["maxpool_c%d_mb" % c])
        y = agg((s, n))
        assert rel_err(y.cpu().numpy(), g["maxpool_c%d_out" % c]) < TOL
    agg = gs.GCNAggregator(50, 16)
    assert set(agg.vars) == {"weights"}
    _inject(agg, weights=g["gcn_w"])
    assert rel_err(agg((s, n)).cpu().numpy(), g["gcn_out"]) < TOL
    agg = gs.MeanAggregator(50, 16, neigh_input_dim=24, act=lambda x: x, concat=True)
    _inject(agg, neigh_weights=g["mean_id_nw"], self_weights=g["mean_id_sw"])
    assert rel_err(agg((s, dev(g["neigh2"]))).cpu().numpy(), g["mean_id_out"]) < TOL
    gs.set_default_math("fp32")


def test_glorot_range_and_bias(gs):
    w = gs.inits.glorot([602, 128]).cpu().numpy()
    r = oracle.glorot_range((602, 128))
    assert w.dtype == np.float32 and np.abs(w).max() <= r and np.abs(w).max() > 0.99 * r and abs(w.mean()) < 1e-3
    agg = gs.MeanAggregator(8, 4, bias=True, concat=True)      # reference crashes here (appendix A); we support it
    agg.vars["bias"] = dev(np.arange(8, dtype=np.float32))
    x, nb = torch.zeros(3, 8).cuda(), torch.zeros(3, 2, 8).cuda()
    np.testing.assert_allclose(agg((x, nb)).cpu().numpy(), np.tile(np.arange(8, dtype=np.float32), (3, 1)))


# ---------------------------------------------------------------- K-hop recursion (golden)
_KEYMAP = {"neigh_weights": "neigh_weights", "self_weights": "self_weights", "weights": "weights"}


def _build_model(gs, g, model, seed=123, counter=40):
    kind = {"mean": "mean", "mean3": "mean", "gcn": "gcn", "maxpool": "maxpool"}[model]
    fan = [int(x) for x in g[model + "_fanout"]]
    dims = [int(x) for x in g[model + "_dims"]]
    sampler = gs.UniformNeighborSampler(dev(g["adj"]), seed=seed)
    sampler.counter = counter
    infos = [gs.SAGEInfo("node", sampler, fan[i], dims[i + 1]) for i in range(len(fan))]
    m = gs.SampleAndAggregate({"batch_size": len(g["seeds"]), "dropout": 0.}, dev(g["feats"]), dev(g["adj"]), None,
                              infos, concat=bool(g[model + "_concat"]), aggregator_type=kind)
    return m, infos, fan, dims


@pytest.mark.parametrize("math", MATHS)
@pytest.mark.parametrize("model", ["mean", "gcn", "maxpool", "mean3"])
def test_khop_golden(gs, model, math):
    g = load_golden("khop")
    gs.set_default_math(math)
    m, infos, fan, dims = _build_model(gs, g, model)
    samples, support = m.sample(dev(g["seeds"]), infos)
    assert support == [int(x) for x in g[model + "_support"]]
    for h, s in enumerate(samples):
        np.testing.assert_array_equal(s.cpu().numpy(), g["%s_samples%d" % (model, h)])       # bit-exact indices
    out, aggs = m.aggregate(samples, [m.features], dims, fan, support, concat=bool(g[model + "_concat"]))
    # inject the reference's weights, then re-run with the same aggregators (models.py:316-317)
    for li, a in enumerate(aggs):
        for key in list(a.vars):
            _inject(a, **{key: g["%s_L%d_%s" % (model, li, key)]})
        if hasattr(a, "mlp_layers"):
            _inject(a.mlp_layers[0], weights=g["%s_L%d_mlp_weights" % (model, li)],
                    bias=g["%s_L%d_mlp_bias" % (model, li)])
    out, _ = m.aggregate(samples, [m.features], dims, fan, support, aggregators=aggs,
                         concat=bool(g[model + "_concat"]))
    assert rel_err(out.cpu().numpy(), g[model + "_out"]) < TOL
    out_l2 = gs.ops.l2_normalize_rows_(out.clone())
    assert rel_err(out_l2.cpu().numpy(), g[model + "_out_l2"]) < TOL
    # the literal (materialised) recursion gives the same answer as the gather-fused one
    lit = m._aggregate_materialised(samples, m.features, dims, fan, support, len(g["seeds"]), aggs,
                                    bool(g[model + "_concat"]))
    assert rel_err(lit.cpu().numpy(), g[model + "_out"]) < TOL
    gs.set_default_math("fp32")


# ---------------------------------------------------------------- full-size Reddit shape (BASELINE configs[1])
@pytest.fixture(scope="module")
def reddit(gs):
    from graphsage_b200.synthetic import reddit_like
    g = reddit_like(n=232965, f=602, max_degree=128, seed=123)
    P = gs.ops.pad_cols(602)
    table = torch.zeros((g["n"] + 1, P), dtype=torch.float32, device="cuda")
    table[:, :602] = torch.from_numpy(g["features"]).cuda()
    g["table"] = table
    g["adj_dev"] = torch.from_numpy(g["adj"]).cuda()
    return g


@pytest.mark.parametrize("math", MATHS)
@pytest.mark.parametrize("kind,concat,dim", [("mean", True, 128), ("gcn", False, 256)])
def test_full_size_forward_vs_oracle(gs, reddit, kind, concat, dim, math):
    gs.set_default_math(math)
    g = reddit
    rs = np.random.RandomState(1)
    B = 512
    seeds = rs.randint(0, g["n"], size=B).astype(np.int32)
    sampler = gs.UniformNeighborSampler(g["adj_dev"], seed=123)
    infos = [gs.SAGEInfo("node", sampler, 25, dim), gs.SAGEInfo("node", sampler, 10, dim)]
    m = gs.SampleAndAggregate({"batch_size": B, "dropout": 0.}, g["table"][:, :602], g["adj_dev"], None, infos,
                              concat=concat, aggregator_type=kind)
    out = m.forward(torch.from_numpy(seeds), normalize=True)
    assert tuple(out.shape) == (B, 256)
    aggs = []
    for a in m.aggregators:
        d = {"type": kind}
        d.update({k: v.cpu().numpy() for k, v in a.vars.items()})
        aggs.append(d)
    ref = oracle.forward_2hop(g["adj"], g["features"], seeds, [25, 10], aggs, concat, 123, 0, normalize=True)
    assert rel_err(out.cpu().numpy(), ref) < TOL
    assert elem_err(out.cpu().numpy(), ref) < 50 * TOL      # elementwise, small entries judged against 1 % of the row scale
    # size-independent properties: unit rows; sampled ids are members of the adjacency rows
    assert np.allclose(np.linalg.norm(out.cpu().numpy(), axis=1), 1.0, atol=1e-5)
    sampler.counter = 0
    samples, support = m.sample(torch.from_numpy(seeds).cuda(), infos)
    assert [s.numel() for s in samples] == [512, 5120, 128000] and support == [1, 10, 250]
    s1 = samples[1].cpu().numpy().reshape(B, 10)
    s2 = samples[2].cpu().numpy().reshape(B * 10, 25)
    for i in range(0, B, 17):
        assert set(s1[i].tolist()) <= set(g["adj"][seeds[i]].tolist())
    for i in range(0, B * 10, 311):
        assert set(s2[i].tolist()) <= set(g["adj"][s1.reshape(-1)[i]].tolist())
    gs.set_default_math("fp32")


BF16_TOL = 2e-2      # config 3 (bf16 operands, fp32 accumulate) vs the fp32 oracle; SURVEY section 7's stated bf16 tolerance


def test_full_size_maxpool_bf16_vs_oracle(gs, reddit):
    """BASELINE configs[2] at its own size: bf16 feature table, K4 (wgmma) for both layers' MLPs, against
    oracle.forward_2hop (reference aggregators.py:168-195) - once on the fp32 operands (bf16 tolerance) and once on the
    bf16-rounded feature table + MLP weights (what K4 multiplies), where only layer 1's activation cast is left."""
    gs.set_default_math("bf16")
    g = reddit
    rs = np.random.RandomState(2)
    B = 512
    seeds = rs.randint(0, g["n"], size=B).astype(np.int32)
    table = g["table"].to(torch.bfloat16)
    sampler = gs.UniformNeighborSampler(g["adj_dev"], seed=123)
    infos = [gs.SAGEInfo("node", sampler, 25, 128), gs.SAGEInfo("node", sampler, 10, 128)]
    m = gs.SampleAndAggregate({"batch_size": B, "dropout": 0.}, table[:, :602], g["adj_dev"], None, infos,
                              concat=True, aggregator_type="maxpool")
    gs.ops.LAUNCHES = 0
    out = m.forward(torch.from_numpy(seeds), normalize=True)
    # second forward on the same model with OTHER seeds (ADVICE r1: the layer-1 bf16 source must not be cached)
    seeds2 = rs.randint(0, g["n"], size=B).astype(np.int32)
    out2 = m.forward(torch.from_numpy(seeds2), normalize=True)
    torch.cuda.synchronize()
    assert tuple(out.shape) == (B, 256)
    aggs, aggs_r = [], []
    for a in m.aggregators:
        d = {"type": "maxpool", "mlp_weights": a.mlp_layers[0].vars["weights"].cpu().numpy(),
             "mlp_bias": a.mlp_layers[0].vars["bias"].cpu().numpy()}
        d.update({k: v.cpu().numpy() for k, v in a.vars.items()})
        aggs.append(d)
        aggs_r.append(dict(d, mlp_weights=bf16_round(d["mlp_weights"])))
    for sd, o, c0 in ((seeds, out, 0), (seeds2, out2, 2)):
        ref = oracle.forward_2hop(g["adj"], g["features"], sd, [25, 10], aggs, True, 123, c0, normalize=True)
        assert rel_err(o.cpu().numpy(), ref) < BF16_TOL
        ref_r = oracle.forward_2hop(g["adj"], bf16_round(g["features"]), sd, [25, 10], aggs_r, True, 123, c0, normalize=True)
        assert rel_err(o.cpu().numpy(), ref_r) < BF16_TOL / 2
        assert np.allclose(np.linalg.norm(o.cpu().numpy(), axis=1), 1.0, atol=1e-5)
    gs.set_default_math("fp32")


def test_maxpool_bf16_eager_steps_do_not_alias(gs):
    """Two different batches through ONE eager bf16 max-pool model: each must equal a fresh model's answer bit for bit
    (the layer-1 source is a fresh torch.empty buffer with a recycled address every step)."""
    rs = np.random.RandomState(13)
    n, f, B = 600, 602, 64
    adj = rs.randint(0, n, size=(n + 1, 32)).astype(np.int32)
    adj[n] = n
    feats = dev(np.vstack([rs.randn(n, f).astype(np.float32), np.zeros((1, f), np.float32)])).to(torch.bfloat16)
    table = torch.zeros((n + 1, gs.ops.pad_cols(f)), dtype=torch.bfloat16, device="cuda")
    table[:, :f] = feats
    batches = [rs.randint(0, n, size=B).astype(np.int32) for _ in range(3)]
    gs.set_default_math("bf16")

    def make():
        gs.inits.manual_seed(11)
        sampler = gs.UniformNeighborSampler(dev(adj), seed=5)
        infos = [gs.SAGEInfo("node", sampler, 25, 128), gs.SAGEInfo("node", sampler, 10, 128)]
        return gs.SampleAndAggregate({"batch_size": B, "dropout": 0.}, table[:, :f], dev(adj), None, infos, concat=True,
                                     aggregator_type="maxpool"), sampler

    m, _ = make()
    got = [m.forward(dev(b), normalize=True).clone() for b in batches]
    for i, b in enumerate(batches):
        fresh, smp = make()
        smp.counter = 2 * i
        assert torch.equal(fresh.forward(dev(b), normalize=True), got[i]), "eager step %d aliases an earlier step" % i
    gs.set_default_math("fp32")


def test_gather_rows_f32_and_cast_rows_bf16(gs):
    rs = np.random.RandomState(21)
    n_rows, F = 700, 602
    x = rs.randn(n_rows, F).astype(np.float32)
    P = gs.ops.pad_cols(F)
    tb = torch.full((n_rows, P), 7.0, dtype=torch.bfloat16, device="cuda")
    tb[:, :F] = dev(x).to(torch.bfloat16)
    ids = rs.randint(-2, n_rows + 3, size=333).astype(np.int32)
    clamp = np.where((ids < 0) | (ids >= n_rows), n_rows - 1, ids)
    out = gs.ops.gather_rows_f32(tb[:, :F], ids=dev(ids))
    assert out.dtype == torch.float32 and out.stride(0) == P
    np.testing.assert_array_equal(out.cpu().numpy(), bf16_round(x)[clamp])
    assert float(out.as_strided((333, P), (P, 1))[:, F:].abs().max()) == 0.0          # pad columns zeroed
    out = gs.ops.gather_rows_f32(dev(x), row0=10, n=50)
    np.testing.assert_array_equal(out.cpu().numpy(), x[10:60])
    c = gs.ops.cast_rows_bf16(dev(x))
    assert c.dtype == torch.bfloat16 and c.stride(0) == P
    np.testing.assert_array_equal(c.float().cpu().numpy(), bf16_round(x))
    assert float(c.as_strided((n_rows, P), (P, 1))[:, F:].float().abs().max()) == 0.0
    sp = torch.tensor([[float("nan"), float("inf"), -float("inf"), 3.0e38, 1e-40, -0.0, 1.0, 2.0]], device="cuda")
    got = gs.ops.cast_rows_bf16(sp).float().cpu().numpy()
    want = sp.to(torch.bfloat16).float().cpu().numpy()
    assert np.array_equal(np.isnan(got), np.isnan(want)) and np.array_equal(got[~np.isnan(got)], want[~np.isnan(want)])


def test_maxpool_step_launches_only_library_kernels(gs):
    """config 3's step must consist of the library's kernels only: count torch-side device work with the profiler."""
    g = load_golden("khop")
    rs = np.random.RandomState(3)
    n, f, B = 300, 602, 64
    adj = g["adj"][:, :32]
    table = torch.zeros((n + 1, gs.ops.pad_cols(f)), dtype=torch.bfloat16, device="cuda")
    table[:n, :f] = dev(rs.randn(n, f).astype(np.float32)).to(torch.bfloat16)
    gs.set_default_math("bf16")
    sampler = gs.UniformNeighborSampler(dev(adj), seed=5)
    infos = [gs.SAGEInfo("node", sampler, 25, 128), gs.SAGEInfo("node", sampler, 10, 128)]
    m = gs.SampleAndAggregate({"batch_size": B, "dropout": 0.}, table[:, :f], dev(adj), None, infos, concat=True,
                              aggregator_type="maxpool")
    seeds = dev(rs.randint(0, n, size=B).astype(np.int32))
    m.forward(seeds, normalize=True)                      # creates aggregators, packs weights
    torch.cuda.synchronize()
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        m.forward(seeds, normalize=True)
        torch.cuda.synchronize()
    gs.set_default_math("fp32")
    names = [e.name for e in prof.events() if e.device_type == DeviceType.CUDA]
    if not names:
        pytest.skip("the profiler recorded no device activity here (CUPTI unavailable)")
    foreign = [nm for nm in names if "gs::" not in nm and "memcpy" not in nm.lower() and "memset" not in nm.lower()]
    assert any("maxpool_mlp" in nm for nm in names), names
    assert not foreign, "non-library kernels in the max-pool step: %r" % foreign


def test_full_size_gather_checksum(gs, reddit):
    g = reddit
    rs = np.random.RandomState(4)
    ids = rs.randint(0, g["n"] + 1, size=133632).astype(np.int32)     # one batch's 512*(1+10+250) rows
    out = gs.ops.gather_rows(g["table"], dev(ids))
    ref = g["table"][dev(ids).long()]
    assert torch.equal(out, ref)
    # gathering is linear in the table: gather(a*T) == a*gather(T) exactly for a power of two
    out2 = gs.ops.gather_rows(g["table"] * 2.0, dev(ids))
    assert torch.equal(out2, out * 2.0)


def test_graphed_forward_matches_eager_and_oracle(gs):
    g = load_golden("khop")
    m, infos, fan, dims = _build_model(gs, g, "mean", counter=40)
    B = len(g["seeds"])
    seeds = dev(g["seeds"])
    eager0 = m.forward(seeds, normalize=True).clone()          # counters 40, 41
    eager1 = m.forward(seeds, normalize=True).clone()          # counters 42, 43
    infos[0].neigh_sampler.counter = 40
    runner = m.graphed(B, normalize=True, probe="gather_mean/%d" % (B * (1 + fan[1])))
    assert len(runner.graphs) == 3 and runner.probe_index == 1
    ev = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
    r0 = runner(seeds, probe_events=ev).clone()
    r1 = runner(seeds).clone()
    torch.cuda.synchronize()
    assert ev[0].elapsed_time(ev[1]) > 0
    assert torch.equal(r0, eager0) and torch.equal(r1, eager1)
    runner.reset(0)
    assert torch.equal(runner(seeds), eager0)
    # replay from pinned host ids
    assert torch.equal(runner(torch.from_numpy(g["seeds"]).pin_memory()), eager1)
    runner.close()


# ---------------------------------------------------------------- tensor-core GEMM (all math modes) vs fp64
GEMM_TOL = {"fp32": 2e-6, "tf32x3": 2e-5, "tf32": 3e-3, "bf16": 2e-2}


@pytest.mark.parametrize("math", ["fp32", "tf32x3", "tf32", "bf16"])
@pytest.mark.parametrize("shape", [
    # (M, [(K, N), ...], combine, bias, act)
    (5632, [(602, 128), (602, 128)], "concat", False, True),      # mean layer 0 at bench size
    (512, [(256, 128), (256, 128)], "concat", False, False),      # mean layer 1
    (5632, [(602, 256)], "add", False, True),                     # gcn layer 0
    (300, [(50, 16), (24, 16)], "add", True, True),               # small, ragged, two K's summed
    (1000, [(602, 512)], "add", True, True),                      # max-pool MLP Dense (bias + relu), 4 N tiles
    (129, [(33, 200), (7, 40)], "concat", True, False),           # nothing aligned
    (1, [(8, 8)], "add", False, False),
])
def test_sage_gemm_math_modes(gs, math, shape):
    M, kn, combine, use_bias, relu = shape
    rs = np.random.RandomState(M + len(kn))
    code = gs.aggregators._MATH_NAMES[math]
    parts, ref_parts = [], []
    for (K, N) in kn:
        lda = gs.ops.pad_cols(K) if K % 2 == 0 else K                 # exercise both aligned and unaligned pitches
        A = torch.zeros((M, lda), dtype=torch.float32, device="cuda")
        a = rs.randn(M, K).astype(np.float32)
        A[:, :K] = dev(a)
        if lda > K:
            A[:, K:] = 1e30                                             # pad columns must never be read
        B = (rs.randn(K, N) / np.sqrt(K)).astype(np.float32)
        parts.append((A, K, dev(B)))
        ref_parts.append(a.astype(np.float64) @ B.astype(np.float64))
    ntot = sum(n for _, n in kn) if combine == "concat" else kn[0][1]
    bias = rs.randn(ntot).astype(np.float32) if use_bias else None
    ref = np.concatenate(ref_parts, axis=1) if combine == "concat" else sum(ref_parts)
    if use_bias:
        ref = ref + bias
    if relu:
        ref = np.maximum(ref, 0)
    out = gs.ops.sage_gemm(parts, combine=gs.ops.COMBINE_CONCAT if combine == "concat" else gs.ops.COMBINE_ADD,
                           bias=None if bias is None else dev(bias), act=gs.ops.ACT_RELU if relu else gs.ops.ACT_NONE,
                           math=code)
    torch.cuda.synchronize()
    assert tuple(out.shape) == (M, ntot)
    assert rel_err(out.cpu().numpy(), ref) < GEMM_TOL[math], (math, shape)


# ---------------------------------------------------------------- fused step kernels
def test_khop_sampler_equals_successive_calls(gs):
    rs = np.random.RandomState(8)
    n, md = 5000, 128
    adj = rs.randint(0, n, size=(n + 1, md)).astype(np.int32)
    adj[n] = n
    seeds = rs.randint(0, n + 1, size=512).astype(np.int32)
    for fan in ([10, 25], [3], [4, 3, 2], [64, 2]):
        outs = gs.ops.sample_padded_khop(dev(adj), dev(seeds), fan, 123, 7)
        cur, cnt = seeds, 7
        for k, o in zip(fan, outs):
            cur = oracle.sample_padded(adj, cur, k, 123, cnt).reshape(-1)
            np.testing.assert_array_equal(o.cpu().numpy(), cur)
            cnt += 1
    cdev = torch.tensor([5], dtype=torch.int64).cuda()
    outs = gs.ops.sample_padded_khop(dev(adj), dev(seeds), [10, 25], 123, 2, counter_dev=cdev)
    np.testing.assert_array_equal(outs[0].cpu().numpy(), oracle.sample_padded(adj, seeds, 10, 123, 7).reshape(-1))
    with pytest.raises(RuntimeError, match="fanout"):
        gs.ops.sample_padded_khop(dev(adj), dev(seeds), [65], 1, 1)


@pytest.mark.parametrize("kind", ["mean_concat", "mean_add", "gcn"])
def test_small_layer_matches_generic_path(gs, kind):
    rs = np.random.RandomState(12)
    B, k, F, D = 301, 10, 256, 128
    H = dev(rs.randn(B + B * k, F).astype(np.float32))
    seg = [gs.ops.Seg(B, k, self_row0=0, neigh_row0=B)]
    bias = dev(rs.randn(2 * D if kind == "mean_concat" else D).astype(np.float32))
    if kind == "gcn":
        agg = gs.GCNAggregator(F, D, bias=True)
    else:
        agg = gs.MeanAggregator(F, D, concat=(kind == "mean_concat"), bias=True)
    agg.vars["bias"] = bias
    final = {"l2_normalize": True, "bump": (torch.zeros(1, dtype=torch.int64).cuda(), 3)}
    fused = agg.aggregate_rows(H, seg, final=final)
    assert final["normalized"] and final["bumped"] and int(final["bump"][0].item()) == 3
    old = gs.ops.SMALL_LAYER_MAX_ROWS
    gs.ops.SMALL_LAYER_MAX_ROWS = 0
    try:
        generic = gs.ops.l2_normalize_rows_(agg.aggregate_rows(H, seg).contiguous())
    finally:
        gs.ops.SMALL_LAYER_MAX_ROWS = old
    assert rel_err(fused.cpu().numpy(), generic.cpu().numpy()) < 2e-6
    # and against numpy
    h = H.cpu().numpy()
    selfv, neigh = h[:B], h[B:].reshape(B, k, F)
    if kind == "gcn":
        ref = oracle.gcn_aggregator(selfv, neigh, agg.vars["weights"].cpu().numpy(), act=lambda x: x) + bias.cpu().numpy()
    else:
        ref = oracle.mean_aggregator(selfv, neigh, agg.vars["neigh_weights"].cpu().numpy(),
                                     agg.vars["self_weights"].cpu().numpy(), concat=(kind == "mean_concat"),
                                     act=lambda x: x) + bias.cpu().numpy()
    ref = oracle.l2_normalize(np.maximum(ref, 0))
    assert rel_err(fused.cpu().numpy(), ref) < 1e-5


def test_packed_weights_follow_weight_updates(gs):
    gs.set_default_math("tf32x3")
    try:
        agg = gs.MeanAggregator(64, 32, concat=True)
        x, nb = torch.randn(200, 64).cuda(), torch.randn(200, 5, 64).cuda()
        y0 = agg((x, nb)).clone()
        agg.vars["self_weights"].mul_(2.0)                      # in-place update must trigger a re-pack
        y1 = agg((x, nb))
        assert rel_err(y1[:, :32].cpu().numpy(), np.maximum(2.0 * (x @ (agg.vars["self_weights"] / 2)).cpu().numpy(), 0)) < 1e-4
        assert torch.equal(y1[:, 32:], y0[:, 32:])
        agg.vars["neigh_weights"] = torch.zeros_like(agg.vars["neigh_weights"])   # replacement too
        assert float(agg((x, nb))[:, 32:].abs().max()) == 0.0
    finally:
        gs.set_default_math("fp32")


# ---------------------------------------------------------------- K4: fused max-pool MLP (bf16 wgmma)
@pytest.mark.parametrize("case", [
    # (n_groups, k, K, hidden, use_ids)
    (5120, 25, 602, 512, True),        # bench shape, hop 2 of layer 0 (one 10th of it)
    (517, 10, 602, 512, True),         # ragged group count, 12 groups per tile
    (301, 10, 256, 512, False),        # layer 1: dense row ranges, 4 K-blocks
    (40, 7, 50, 128, True),            # small K (one partial K-block), one hidden slice
    (3, 128, 64, 256, True),           # one group per tile
    (1000, 1, 602, 1024, True),        # k = 1 (max over a single row), "big" hidden
])
@pytest.mark.parametrize("variant", ["tmem128c", "tmem128c2", "tmem128", "tmem128x2", "tmem256", "wide128_tma", "wide128_cpasync", "wide256_cpasync", "round1"])
def test_maxpool_mlp_fused_vs_reference(gs, case, variant):
    n_groups, k, K, hidden, use_ids = case
    if k > K4_VARIANTS[variant][1]:
        pytest.skip("fanout %d needs a wider tile than %d" % (k, K4_VARIANTS[variant][1]))
    _k4_select(gs, variant)
    try:
        _maxpool_mlp_case(gs, n_groups, k, K, hidden, use_ids)
    finally:
        _k4_select(gs, K4_DEFAULT)


# name -> (k4_operands, k4_tile, k4_mma_depth, k4_producer, k4_cluster): the Hopper kernel configuration each named variant
# runs (maxpool_tc.cu).  k4_operands 1 = gathered rows are the wgmma A operand, 0 = the weight slice is A and the rows are
# B; k4_tile = rows per tile; k4_mma_depth = wgmma groups in flight; k4_producer 0 = cp.async row pieces, 1 = register-
# staged 128-bit loads; k4_cluster = thread-block cluster of a tile's hidden slices (-1 = all of them, 0 = none).
K4_VARIANTS = {"tmem128c2": (0, 128, 1, 0, 2),        # weights as A, PAIRS of a tile's hidden slices form a cluster
               "tmem128c": (0, 128, 1, 0, -1),        # weights as A, clusters of all hidden/128 slices of a tile
               "tmem128": (0, 128, 1, 0, 0),          # weights as A, no clusters
               "tmem128x2": (0, 128, 2, 0, 0),        # weights as A, two wgmma groups in flight
               "tmem256": (0, 256, 1, 0, 0),          # weights as A, 256-row tiles (N = 2 x 128 per K step)
               "wide128_tma": (0, 128, 1, 1, 0),      # weights as A, register-staged row loads
               "wide128_cpasync": (1, 128, 2, 0, 0),  # rows as A, two wgmma groups in flight
               "wide256_cpasync": (1, 256, 1, 0, 0),  # rows as A, 256-row tiles (two m64 blocks per warpgroup)
               "round1": (1, 128, 1, 0, 0)}           # rows as A, 128-row tiles: the default
K4_DEFAULT = "round1"


def _k4_select(gs, name):
    operands, tile, depth, producer, cluster = K4_VARIANTS[name]
    gs._lib.set_tuning("k4_operands", operands)
    gs._lib.set_tuning("k4_tile", tile)
    gs._lib.set_tuning("k4_mma_depth", depth)
    gs._lib.set_tuning("k4_producer", producer)
    gs._lib.set_tuning("k4_cluster", cluster)


def test_maxpool_mlp_fused_wide_fanouts(gs):
    """ragged last tiles, one group per tile, single-K-block tiles, odd tile counts, K with / without a partial last
    K-block, fanouts above 128 (256-row tiles only); a fanout above the tile is refused"""
    cases = ((7, 128, 602, 128), (1, 25, 602, 512), (2049, 3, 96, 128), (11, 100, 300, 128), (3, 33, 640, 256),
             (900, 5, 64, 128), (333, 7, 33, 128), (260, 25, 512, 256), (260, 25, 513, 128), (1500, 25, 602, 128))
    wide = ((7, 200, 602, 128), (2, 256, 64, 256), (11, 129, 300, 128), (700, 9, 32, 128))
    try:
        for name in ("tmem128c", "tmem128c2", "tmem128", "tmem128x2", "tmem256", "wide128_tma", "wide128_cpasync", "wide256_cpasync"):
            _k4_select(gs, name)
            tile = K4_VARIANTS[name][1]
            for case in cases + (wide if tile == 256 else ()):
                _maxpool_mlp_case(gs, *case, True)
            with pytest.raises(RuntimeError, match="k <= %d" % tile):
                _maxpool_mlp_case(gs, 2, tile + 1, 64, 128, True)
    finally:
        _k4_select(gs, K4_DEFAULT)


def _maxpool_mlp_case(gs, n_groups, k, K, hidden, use_ids):
    rs = np.random.RandomState(n_groups + k)
    n_rows = 4000
    P = gs.ops.pad_cols(K)
    table = torch.zeros((n_rows, P), dtype=torch.bfloat16, device="cuda")
    table[:, :K] = dev(rs.randn(n_rows, K).astype(np.float32)).to(torch.bfloat16)
    if P > K:
        table[:, K:] = 3.0                                      # pad columns must not leak into the result
    W = dev((rs.randn(K, hidden) / np.sqrt(K)).astype(np.float32))
    bias = dev(rs.randn(hidden).astype(np.float32))
    packed = gs.ops.PackedMlpWeights()
    if use_ids:
        ids = rs.randint(0, n_rows, size=n_groups * k).astype(np.int32)
        out = gs.ops.maxpool_mlp_fused(table[:, :K], n_groups, k, W, bias, packed, row_ids=dev(ids))
        rows = table[dev(ids).long(), :K].float()
    else:
        row0 = 100
        out = gs.ops.maxpool_mlp_fused(table[:, :K], n_groups, k, W, bias, packed, row0=row0)
        rows = table[row0:row0 + n_groups * k, :K].float()
    torch.cuda.synchronize()
    assert tuple(out.shape) == (n_groups, hidden)
    # the oracle's neighbour branch (reference aggregators.py:176-182: Dense(relu, bias) -> reduce_max) on the SAME
    # bf16-rounded operands, in fp64 and in the oracle's own fp32: identity self/neigh weights isolate the branch
    neigh = rows.cpu().numpy().reshape(n_groups, k, K)
    Wr = bf16_round(W.cpu().numpy())
    eye = np.eye(hidden)
    zero_self = np.zeros((n_groups, 1))
    ref64 = oracle.maxpool_aggregator(zero_self, neigh.astype(np.float64), Wr.astype(np.float64),
                                      bias.cpu().numpy().astype(np.float64), eye, np.zeros((1, hidden)), concat=False,
                                      act=lambda x: x)
    assert rel_err(out.cpu().numpy(), ref64) < 2e-5                  # same bf16 operands, fp32 accumulate
    ref32 = oracle.maxpool_aggregator(zero_self.astype(np.float32), neigh, Wr, bias.cpu().numpy(), eye.astype(np.float32),
                                      np.zeros((1, hidden), np.float32), concat=False, act=lambda x: x)
    assert rel_err(out.cpu().numpy(), ref32) < TOL


def test_maxpool_bf16_model_matches_fp32_model(gs):
    """config 3 (bf16 max-pool path through K4) vs the fp32 generic path on the same weights: bf16-level agreement."""
    g = load_golden("khop")
    rs = np.random.RandomState(3)
    n, f, B = 300, 602, 64
    adj = g["adj"][:, :32]
    feats = np.vstack([rs.randn(n, f).astype(np.float32), np.zeros((1, f), np.float32)])
    seeds = rs.randint(0, n, size=B).astype(np.int32)
    outs = {}
    for math, table in (("fp32", dev(feats)), ("bf16", dev(feats).to(torch.bfloat16))):
        gs.set_default_math(math)
        gs.inits.manual_seed(11)
        sampler = gs.UniformNeighborSampler(dev(adj), seed=5)
        infos = [gs.SAGEInfo("node", sampler, 25, 128), gs.SAGEInfo("node", sampler, 10, 128)]
        m = gs.SampleAndAggregate({"batch_size": B, "dropout": 0.}, table, dev(adj), None, infos, concat=True,
                                  aggregator_type="maxpool")
        outs[math] = m.forward(dev(seeds), normalize=True).cpu().numpy()
    gs.set_default_math("fp32")
    assert rel_err(outs["bf16"], outs["fp32"]) < 3e-2


def test_pipelined_forward_matches_eager(gs):
    g = load_golden("khop")
    m, infos, fan, dims = _build_model(gs, g, "mean", counter=40)
    B = len(g["seeds"])
    rs = np.random.RandomState(4)
    n = g["adj"].shape[0] - 1
    batches = [rs.randint(0, n, size=B).astype(np.int32) for _ in range(5)]
    eager = [m.forward(dev(b), normalize=True).clone() for b in batches]        # counters 40.. 49
    infos[0].neigh_sampler.counter = 40
    pipe = m.pipelined(B)
    ids_host = [torch.from_numpy(b).pin_memory() for b in batches]
    outs = [torch.empty((B, eager[0].shape[1]), dtype=torch.float32).pin_memory() for _ in batches]
    for i in range(5):
        pipe.submit(ids_host[i], outs[i])
    pipe.synchronize()
    for i in range(5):
        assert torch.equal(outs[i], eager[i].cpu()), "pipelined step %d differs from eager step %d" % (i, i)
    # a short (last, partial) id batch or a wrong result buffer must raise, not read past the host buffer
    with pytest.raises(ValueError, match="batch size"):
        pipe.submit(ids_host[0][:B - 1], outs[0])
    with pytest.raises(ValueError, match="out_host"):
        pipe.submit(ids_host[0], outs[0].double())
    pipe.close()


# ---------------------------------------------------------------- mean-pool aggregator (SURVEY 8f row 4)
def test_meanpool_golden_and_fused(gs):
    g = load_golden("meanpool")
    s, n = dev(g["self"]), dev(g["neigh"])
    gs.set_default_math("fp32")
    for c in (0, 1):
        agg = gs.MeanPoolingAggregator(40, 16, concat=bool(c))
        assert agg.hidden_dim == 512 and agg.pool == "mean"
        _inject(agg, neigh_weights=g["c%d_nw" % c], self_weights=g["c%d_sw" % c])
        _inject(agg.mlp_layers[0], weights=g["c%d_mw" % c], bias=g["c%d_mb" % c])
        assert rel_err(agg((s, n)).cpu().numpy(), g["c%d_out" % c]) < TOL
    # K4 with the mean epilogue vs an fp64 reference on the same bf16 operands
    rs = np.random.RandomState(6)
    n_rows, K, hidden, n_groups, k = 3000, 602, 512, 777, 25
    table = torch.zeros((n_rows, gs.ops.pad_cols(K)), dtype=torch.bfloat16, device="cuda")
    table[:, :K] = dev(rs.randn(n_rows, K).astype(np.float32)).to(torch.bfloat16)
    W = dev((rs.randn(K, hidden) / np.sqrt(K)).astype(np.float32))
    bias = dev(rs.randn(hidden).astype(np.float32))
    ids = rs.randint(0, n_rows, size=n_groups * k).astype(np.int32)
    out = gs.ops.maxpool_mlp_fused(table[:, :K], n_groups, k, W, bias, gs.ops.PackedMlpWeights(), row_ids=dev(ids),
                                   pool="mean")
    rows = table[dev(ids).long(), :K].double()
    ref = torch.relu(rows @ W.to(torch.bfloat16).double() + bias.double()).reshape(n_groups, k, hidden).mean(dim=1)
    assert rel_err(out.cpu().numpy(), ref.cpu().numpy()) < 2e-5
    # and through the model: aggregator_type="meanpool"
    gk = load_golden("khop")
    sampler = gs.UniformNeighborSampler(dev(gk["adj"]), seed=3)
    infos = [gs.SAGEInfo("node", sampler, 4, 8), gs.SAGEInfo("node", sampler, 2, 8)]
    m = gs.SampleAndAggregate({"batch_size": 9, "dropout": 0.}, dev(gk["feats"]), dev(gk["adj"]), None, infos,
                              concat=True, aggregator_type="meanpool")
    emb = m.export_embeddings(np.arange(20), batch_size=9)
    assert emb.shape == (20, 16) and np.allclose(np.linalg.norm(emb, axis=1), 1.0, atol=1e-5)


# ---------------------------------------------------------------- device-side padded adjacency (SURVEY 8f row 3)
def test_build_padded_adj_bit_exact(gs):
    from graphsage_b200.synthetic import community_graph_csr
    indptr, indices, comm = community_graph_csr(3000, n_comm=5, mean_deg=20, seed=4)
    rs = np.random.RandomState(1)
    skip = rs.rand(3000) < 0.1
    for md in (16, 25, 128):
        adj, deg = gs.ops.build_padded_adj(dev(indptr), dev(indices), md, seed=123, counter=3, skip=dev(skip))
        ref_adj, ref_deg = oracle.build_padded_adj(indptr, indices, md, 123, 3, skip=skip)
        np.testing.assert_array_equal(adj.cpu().numpy(), ref_adj)
        np.testing.assert_array_equal(deg.cpu().numpy(), ref_deg)
        a = adj.cpu().numpy()
        assert (a[3000] == 3000).all() and (a[np.nonzero(skip)[0]] == 3000).all()
        d = np.diff(indptr)
        for u in np.nonzero((d > md) & ~skip)[0][:50]:
            assert len(set(a[u].tolist())) == md                       # without replacement
            assert set(a[u].tolist()) <= set(indices[indptr[u]:indptr[u + 1]].tolist())
    # the table feeds the sampler directly
    out = gs.ops.sample_padded(adj, dev(np.arange(100, dtype=np.int32)), 10, 1, 1)
    assert out.shape == (100, 10)


# ---------------------------------------------------------------- config 5 pieces: device R-MAT generator, CSR-sampled model
@pytest.mark.parametrize("scale,n", [(13, 5000), (10, 1024), (12, 4095)])
def test_rmat_generator_bit_exact(gs, scale, n):
    from graphsage_b200.synthetic import rmat_csr_device
    ref_ptr, ref_idx = oracle.rmat.rmat_csr(scale, n, 20.0, seed=11)
    for threshold in (4096, 50):                       # 50: the hub rows take the whole-grid path
        indptr, indices = rmat_csr_device(scale, n, 20.0, seed=11, long_threshold=threshold)
        np.testing.assert_array_equal(indptr.cpu().numpy(), ref_ptr)
        np.testing.assert_array_equal(indices.cpu().numpy(), ref_idx)


def test_rmat_generator_properties_at_scale(gs):
    """size-independent properties at a size the oracle would not finish quickly: 2^20 nodes, ~21 M entries"""
    from graphsage_b200.synthetic import rmat_csr_device
    n = 1 << 20
    indptr, indices = rmat_csr_device(20, n, 20.0, seed=123)
    deg = (indptr[1:] - indptr[:-1])
    m = int(indptr[-1])
    assert indices.numel() == m and abs(m / float(n) - 20.0) < 0.1
    assert int(indices.min()) >= 0 and int(indices.max()) < n
    rows = torch.repeat_interleave(torch.arange(n, device="cuda"), deg)
    assert int((rows == indices.long()).sum()) == 0                         # no self loops
    indeg = torch.bincount(indices.long(), minlength=n)
    # b == c: the in-degree and out-degree distributions have the same heavy tail
    assert 0.5 < float(indeg.max()) / float(deg.max()) < 2.0 and int(deg.max()) > 2000
    # the hubs are scrambled over the id range, not packed at its start
    top = torch.topk(deg, 64).indices
    assert int((top < n // 8).sum()) < 32


def test_csr_sampled_model_vs_oracle(gs):
    """SampleAndAggregate over a CSRNeighborSampler (the config-5 path) against the oracle: per-node draws bit-exact
    (oracle.sample_csr), outputs within 1e-4."""
    rs = np.random.RandomState(17)
    indptr, indices = oracle.rmat.rmat_csr(11, 2000, 12.0, seed=3)
    n, f, B = 2000, 64, 96
    feats = np.vstack([rs.randn(n, f).astype(np.float32), np.zeros((1, f), np.float32)])
    seeds = rs.randint(0, n, size=B).astype(np.int32)
    gs.set_default_math("fp32")
    sampler = gs.CSRNeighborSampler(dev(indptr), dev(indices), seed=9)
    infos = [gs.SAGEInfo("node", sampler, 25, 32), gs.SAGEInfo("node", sampler, 10, 32)]
    m = gs.SampleAndAggregate({"batch_size": B, "dropout": 0.}, dev(feats), None, None, infos, concat=True,
                              aggregator_type="mean")
    out = m.forward(dev(seeds), normalize=True).cpu().numpy()
    h1 = oracle.sample_csr(indptr, indices, seeds, 10, 9, 0, pad_id=n).reshape(-1)
    h2 = oracle.sample_csr(indptr, indices, h1, 25, 9, 1, pad_id=n).reshape(-1)
    sampler.counter = 0
    got, support = m.sample(dev(seeds), infos)
    np.testing.assert_array_equal(got[1].cpu().numpy(), h1)
    np.testing.assert_array_equal(got[2].cpu().numpy(), h2)
    aggs = [dict(type="mean", **{k: v.cpu().numpy() for k, v in a.vars.items()}) for a in m.aggregators]
    ref = oracle.l2_normalize(oracle.aggregate_khop([seeds, h1, h2], feats, [25, 10], [1, 10, 250], B, aggs, True))
    assert rel_err(out, ref) < TOL


# ---------------------------------------------------------------- tf32x3 mean / GCN layer with bias on the generic path
@pytest.mark.parametrize("kind", ["mean_concat", "mean_add", "gcn"])
@pytest.mark.parametrize("shape", [(5632, 602, 128, True), (301, 50, 16, False), (1000, 256, 40, True), (129, 33, 8, False)])
def test_mean_gcn_layer_tf32x3_vs_oracle(gs, kind, shape):
    """The gather + tf32x3 GEMM layer (bias, relu, id segments, ragged widths) against the oracle."""
    rows, F, D, two_hops = shape
    rs = np.random.RandomState(rows + F)
    n_src = 4000
    table = torch.zeros((n_src + 1, gs.ops.pad_cols(F)), dtype=torch.float32, device="cuda")
    table[:n_src, :F] = dev(rs.randn(n_src, F).astype(np.float32))
    if two_hops:
        n0 = rows // 11
        n1 = rows - n0
        s0 = dev(rs.randint(0, n_src + 1, size=n0).astype(np.int32))
        s1 = dev(rs.randint(0, n_src + 1, size=n1).astype(np.int32))
        s2 = dev(rs.randint(0, n_src + 1, size=n1 * 25).astype(np.int32))
        s1n = dev(rs.randint(0, n_src + 1, size=n0 * 10).astype(np.int32))
        segs = [gs.ops.Seg(n0, 10, self_ids=s0, neigh_ids=s1n, out_row0=0), gs.ops.Seg(n1, 25, self_ids=s1, neigh_ids=s2, out_row0=n0)]
    else:
        segs = [gs.ops.Seg(rows, 7, self_ids=dev(rs.randint(0, n_src, size=rows).astype(np.int32)),
                           neigh_ids=dev(rs.randint(0, n_src, size=rows * 7).astype(np.int32)))]
    gs.set_default_math("tf32x3")
    old_small = gs.ops.SMALL_LAYER_MAX_ROWS
    gs.ops.SMALL_LAYER_MAX_ROWS = 0
    try:
        if kind == "gcn":
            agg = gs.GCNAggregator(F, 2 * D, bias=True)
        else:
            agg = gs.MeanAggregator(F, D, concat=(kind == "mean_concat"), bias=True)
        agg.vars["bias"] = dev(rs.randn(agg.vars["bias"].numel()).astype(np.float32))
        out = agg.aggregate_rows(table[:, :F], segs)
        t = table[:, :F].cpu().numpy()
        ref_rows = []
        for sg in segs:
            selfv = t[sg.self_ids.cpu().numpy()[:sg.n]]
            neigh = t[sg.neigh_ids.cpu().numpy()[:sg.n * sg.k]].reshape(sg.n, sg.k, F)
            if kind == "gcn":
                ref_rows.append(oracle.gcn_aggregator(selfv, neigh, agg.vars["weights"].cpu().numpy(), act=lambda x: x))
            else:
                ref_rows.append(oracle.mean_aggregator(selfv, neigh, agg.vars["neigh_weights"].cpu().numpy(),
                                                       agg.vars["self_weights"].cpu().numpy(), concat=(kind == "mean_concat"),
                                                       act=lambda x: x))
        ref = np.maximum(np.vstack(ref_rows) + agg.vars["bias"].cpu().numpy(), 0)
        assert rel_err(out.cpu().numpy(), ref) < TOL
    finally:
        gs.ops.SMALL_LAYER_MAX_ROWS = old_small
        gs.set_default_math("fp32")


# ---------------------------------------------------------------- bf16 feature table through the fused gather + mean
def test_gather_mean_bf16_table(gs):
    """gs_gather_mean(GS_BF16): fp32 means / self rows from a bfloat16 table - must equal the fp32 kernel on the
    bf16-rounded table bit for bit (same fp32 sums in the same order), for both mean forms, ragged widths and pad columns."""
    rs = np.random.RandomState(31)
    for F, k, n in ((602, 25, 700), (602, 10, 64), (50, 7, 333), (256, 1, 100), (8, 128, 9)):
        n_src = 3000
        P = gs.ops.pad_cols(F)
        x = rs.randn(n_src, F).astype(np.float32)
        tb = torch.full((n_src, P), 5.0, dtype=torch.bfloat16, device="cuda")          # pad columns hold junk
        tb[:, :F] = dev(x).to(torch.bfloat16)
        tf = torch.zeros((n_src, P), dtype=torch.float32, device="cuda")
        tf[:, :F] = tb[:, :F].float()
        seg = [gs.ops.Seg(n, k, self_ids=dev(rs.randint(-1, n_src + 2, size=n).astype(np.int32)),
                          neigh_ids=dev(rs.randint(0, n_src, size=n * k).astype(np.int32)))]
        for include_self in (False, True):
            a = gs.ops.gather_mean(tb[:, :F], seg, include_self=include_self)
            b = gs.ops.gather_mean(tf[:, :F], seg, include_self=include_self)
            assert a[1].dtype == torch.float32 and torch.equal(a[1], b[1]) and torch.equal(a[0], b[0]), (F, k, include_self)
    # and through the model: graphsage_mean over a bf16 table vs the oracle on the rounded features
    g = load_golden("khop")
    n = g["adj"].shape[0] - 1
    feats = np.vstack([rs.randn(n, 602).astype(np.float32), np.zeros((1, 602), np.float32)])
    table = torch.zeros((n + 1, gs.ops.pad_cols(602)), dtype=torch.bfloat16, device="cuda")
    table[:, :602] = dev(feats).to(torch.bfloat16)
    seeds = rs.randint(0, n, size=48).astype(np.int32)
    gs.set_default_math("fp32")
    sampler = gs.UniformNeighborSampler(dev(g["adj"]), seed=4)
    infos = [gs.SAGEInfo("node", sampler, 6, 32), gs.SAGEInfo("node", sampler, 4, 32)]
    m = gs.SampleAndAggregate({"batch_size": 48, "dropout": 0.}, table[:, :602], dev(g["adj"]), None, infos, concat=True,
                              aggregator_type="mean")
    out = m.forward(dev(seeds), normalize=True).cpu().numpy()
    aggs = [dict(type="mean", **{k_: v.cpu().numpy() for k_, v in a.vars.items()}) for a in m.aggregators]
    ref = oracle.forward_2hop(g["adj"], bf16_round(feats), seeds, [6, 4], aggs, True, 4, 0, normalize=True)
    assert rel_err(out, ref) < TOL
