"""CPU: the two-layer max-pool aggregator (TwoMaxLayerPoolingAggregator, aggregator_type="twomaxpool") without a GPU -
the oracle and the aggregator against the reference's own class (tests/golden/twomax.npz: direct calls, a two-layer
sample / aggregate, one dropout pass pinning the mlp -> mlp2 call order and layout), its constructor surface against the
reference's (aggregators.py:276-361), the dropout site plan, the materialised
branch's backward against float64 torch autograd, the autograd wiring of _PoolAggregateRowsFn over two Dense layers
(with and without dropout) with the kernels replaced by torch stand-ins that draw the oracle's masks (TEST mocks only;
the product has no such path), and the refusals."""
import numpy as np
import pytest
import torch

import graphsage_b200 as gs
from graphsage_b200 import ops, supervised_models as sm
from test_dropout_cpu import _tdrop, cpu_kernels  # noqa: F401  (the stand-in kernels fixture)


def test_constructor_surface():
    for size, (h1, h2) in (("small", (512, 256)), ("big", (1024, 512))):
        a = gs.TwoMaxLayerPoolingAggregator(10, 6, model_size=size, device="cpu")
        assert (a.hidden_dim_1, a.hidden_dim_2, a.hidden_dim) == (h1, h2, h2)
        assert sorted(a.vars) == ["neigh_weights", "self_weights"]
        assert tuple(a.vars["neigh_weights"].shape) == (h2, 6) and tuple(a.vars["self_weights"].shape) == (10, 6)
        assert [tuple(l.vars["weights"].shape) for l in a.mlp_layers] == [(10, h1), (h1, h2)]
        assert [tuple(l.vars["bias"].shape) for l in a.mlp_layers] == [(h1,), (h2,)]
        assert all(l.act is gs.relu for l in a.mlp_layers)
        assert isinstance(a, gs.MaxPoolingAggregator) and a.pool == "max"
    a = gs.TwoMaxLayerPoolingAggregator(10, 6, neigh_input_dim=7, dropout=0.3, device="cpu")
    assert a.mlp_layers[0].input_dim == 7 and all(l.dropout == 0.3 for l in a.mlp_layers)
    # bias=True: the reference reads self.output_dim before setting it (a crash); here it is out * (2 if concat)
    for concat, width in ((False, 6), (True, 12)):
        b = gs.TwoMaxLayerPoolingAggregator(10, 6, bias=True, concat=concat, device="cpu")
        assert tuple(b.vars["bias"].shape) == (width,) and not b.vars["bias"].any()
    with pytest.raises(ValueError, match="model_size"):
        gs.TwoMaxLayerPoolingAggregator(10, 6, model_size="medium", device="cpu")
    every, decayed = sm.aggregator_parameters([a])
    assert len(every) == 2 + 4 and len(decayed) == 2
    assert [tuple(t.shape) for t in sm.layer_params(a)] == [(10, 6), (256, 6), (7, 512), (512,), (512, 256), (256,)]
    assert gs.models._AGGREGATORS["twomaxpool"] is gs.TwoMaxLayerPoolingAggregator


def test_dropout_site_plan_adds_mlp2_and_leaves_the_other_kinds_alone():
    assert sm.dropout_site_plan("twomaxpool", 2, head=True) == [
        (0, 0, "mlp"), (0, 0, "mlp2"), (0, 1, "mlp"), (0, 1, "mlp2"), (1, 0, "mlp"), (1, 0, "mlp2"), (None, None, "head")]
    assert sm.dropout_site_plan("maxpool", 2) == [(0, 0, "mlp"), (0, 1, "mlp"), (1, 0, "mlp")]
    assert sm.dropout_site_plan("meanpool", 1, head=True) == [(0, 0, "mlp"), (None, None, "head")]
    assert len(sm.dropout_site_plan("mean", 2)) == 6 and sm.dropout_site_plan("seq", 2) == []


def _ref_layer(selfv, neigh, k, w, sites, concat, last):
    """aggregators.py:330-361 with Dense's input dropout (layers.py:107) in differentiable torch."""
    n = selfv.shape[0]
    d1, d2 = (lambda x: x, lambda x: x) if sites is None else (lambda x: _tdrop(x, sites[0]), lambda x: _tdrop(x, sites[1]))
    h = torch.relu(d1(neigh) @ w["W1"] + w["b1"])
    h = torch.relu(d2(h) @ w["W2"] + w["b2"]).reshape(n, k, -1).amax(dim=1)
    fs, fn = selfv @ w["self_weights"], h @ w["neigh_weights"]
    y = torch.cat([fs, fn], dim=1) if concat else fs + fn
    return y if last else torch.relu(y)


def _params(a):
    w = dict(a.vars)
    for i, layer in enumerate(a.mlp_layers):
        w["W%d" % (i + 1)], w["b%d" % (i + 1)] = layer.vars["weights"], layer.vars["bias"]
    return w


@pytest.mark.parametrize("concat", [True, False])
@pytest.mark.parametrize("rate", [0.0, 0.5])
def test_two_layer_chain_gradients_match_autograd(cpu_kernels, concat, rate):  # noqa: F811
    r = np.random.RandomState(3)
    N, F, d, D, B, k1, k2 = 40, 10, 3, 6, 5, 3, 4
    feats = torch.from_numpy(r.randn(N, F).astype(np.float32))
    feats[7] = 0.0                                       # an all-zero row: every unit ties in the max
    emb = torch.from_numpy(r.randn(N, d).astype(np.float32)).requires_grad_(True)
    table = torch.cat([emb.detach(), feats], dim=1)
    s0 = torch.from_numpy(r.randint(0, N, size=B).astype(np.int32))
    s1 = torch.from_numpy(r.randint(0, N, size=B * k1).astype(np.int32))
    s2 = torch.from_numpy(r.randint(0, N, size=B * k1 * k2).astype(np.int32))
    s2[:k2] = 7
    dim_mult = 2 if concat else 1
    a0 = gs.TwoMaxLayerPoolingAggregator(F + d, D, act=gs.relu, concat=concat, device="cpu")
    a1 = gs.TwoMaxLayerPoolingAggregator(dim_mult * D, D, act=gs.identity, concat=concat, device="cpu")
    params = []
    for a in (a0, a1):
        a.math = ops.MATH_FP32_SIMT
        for layer in a.mlp_layers:
            layer.vars["bias"] = torch.from_numpy(r.randn(layer.output_dim).astype(np.float32) * 0.1)
        for dct in [a.vars] + [layer.vars for layer in a.mlp_layers]:
            for key in dct:
                dct[key] = dct[key].detach().clone().requires_grad_(True)
                params.append(dct[key])
    seed = 99
    sites0 = [((seed, 0, rate), (seed, 1, rate)), ((seed, 2, rate), (seed, 3, rate))] if rate else None
    sites1 = [((seed, 4, rate), (seed, 5, rate))] if rate else None

    def apply(a, src, segs, e, sites):
        return sm._PoolAggregateRowsFn.apply(a, src, segs, *sm.layer_params(a), e, sites)

    seg0 = [ops.Seg(B, k1, self_ids=s0, neigh_ids=s1, out_row0=0), ops.Seg(B * k1, k2, self_ids=s1, neigh_ids=s2, out_row0=B)]
    h1 = apply(a0, table, seg0, emb, sites0)
    out = apply(a1, h1, [ops.Seg(B, k1, self_row0=0, neigh_row0=B, out_row0=0)], None, sites1)
    R = torch.from_numpy(r.randn(*out.shape).astype(np.float32))
    (out * R).sum().backward()
    got = [p.grad.clone() for p in params] + [emb.grad.clone()]
    for p in params + [emb]:
        p.grad = None
    full = torch.cat([emb, feats], dim=1)
    x0, x1, x2 = full[s0.long()], full[s1.long()], full[s2.long()]
    r0 = _ref_layer(x0, x1, k1, _params(a0), sites0 and sites0[0], concat, last=False)
    r1 = _ref_layer(x1, x2, k2, _params(a0), sites0 and sites0[1], concat, last=False)
    ref = _ref_layer(r0, r1, k1, _params(a1), sites1 and sites1[0], concat, last=True)
    assert torch.allclose(out.detach(), ref.detach(), rtol=1e-5, atol=1e-5)
    (ref * R).sum().backward()
    for p, g in zip(params + [emb], got):
        assert p.grad is not None and torch.allclose(g, p.grad, rtol=2e-4, atol=2e-5), float((g - p.grad).abs().max())


def test_branch_backward_matches_fp64_autograd():
    """One hop of the materialised branch's backward (pool_branch_backward for Dense 2, then dpre1 = dh1 [h1 > 0],
    dW1 = x^T dpre1, db1 = sum dpre1, dx = dpre1 W1^T) on float64 operands, ties in the max included."""
    r = np.random.RandomState(1)
    n, k, K, h1w, h2w = 4, 3, 5, 8, 6
    x = torch.from_numpy(r.randn(n * k, K))
    x[0:k] = x[0]                                         # a group of identical rows: k-way ties
    W1, b1, W2, b2 = (torch.from_numpy(r.randn(*s)) for s in ((K, h1w), (h1w,), (h1w, h2w), (h2w,)))
    dhp = torch.from_numpy(r.randn(n, h2w))
    leaves = [t.clone().requires_grad_(True) for t in (x, W1, b1, W2, b2)]
    h1 = torch.relu(leaves[0] @ leaves[1] + leaves[2])
    h2 = torch.relu(h1 @ leaves[3] + leaves[4])
    hp = h2.reshape(n, k, h2w).amax(dim=1)
    (hp * dhp).sum().backward()
    h1d, h2d = h1.detach(), h2.detach()
    dW2, db2, dh1 = sm.pool_branch_backward("max", h1d, h2d, hp.detach(), dhp, W2, k, True)
    dpre1 = dh1 * (h1d > 0).double()
    for got, want in ((dW2, leaves[3]), (db2, leaves[4]), (x.t() @ dpre1, leaves[1]), (dpre1.sum(0), leaves[2]),
                      (dpre1 @ W1.t(), leaves[0])):
        assert torch.allclose(got, want.grad, rtol=1e-12, atol=1e-12)


class _Sampler(object):
    counter, counter_dev = 0, None


def _model(cls=gs.SupervisedGraphsage, **kw):
    N, F = 30, 10
    adj = torch.zeros((N + 1, 8), dtype=torch.int32)
    infos = [gs.SAGEInfo("node", _Sampler(), 4, 8), gs.SAGEInfo("node", _Sampler(), 3, 8)]
    placeholders = {"batch_size": 4, "dropout": 0.}
    args = (placeholders, torch.randn(N + 1, F), adj, np.ones(N), infos)
    if cls is gs.SupervisedGraphsage:
        args = (3,) + args
    return cls(*args, aggregator_type="twomaxpool", device="cpu", **kw)


@pytest.mark.parametrize("cls", [gs.SupervisedGraphsage, gs.UnsupervisedGraphsage])
def test_training_classes_accept_it_and_refuse_the_fused_path(cls):
    m = _model(cls, model_size="big")
    assert all(isinstance(a, gs.TwoMaxLayerPoolingAggregator) and a.hidden_dim_1 == 1024 for a in m.aggregators)
    assert len(m.parameters()) == len(_model(cls).parameters())
    with pytest.raises(NotImplementedError, match="one MLP layer"):
        _model(cls, fused_pool=True)
    with pytest.raises(NotImplementedError, match="twomaxpool"):
        from graphsage_b200.full_neighbor_training import refuse_full_neighbor
        refuse_full_neighbor(m, True)
    from graphsage_b200.full_neighbor_training import refuse_full_neighbor
    refuse_full_neighbor(m, False)                        # inference over whole neighbourhoods is not refused


def test_training_refuses_a_third_dense_layer():
    a = gs.TwoMaxLayerPoolingAggregator(10, 6, device="cpu")
    a.mlp_layers.append(a.mlp_layers[-1])
    with pytest.raises(NotImplementedError, match="one or two MLP layers"):
        sm._PoolAggregateRowsFn(a, [], None).forward(torch.zeros(3, 10), [])


# ---------------------------------------------------------------- pinned against the reference (tests/golden/twomax.npz)
@pytest.fixture(scope="module")
def golden():
    import os
    return dict(np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "twomax.npz")))


def _w(g, key):
    from oracle import pool2_forward as p2
    w = p2.weights_from_draws(g[key + "draws"])
    w.update(b1=g[key + "b1"], b2=g[key + "b2"])
    if key + "bias" in g:
        w["bias"] = g[key + "bias"]
    return w


def _counter_drop(g):
    from oracle import dropout as od
    call = [0]

    def drop(x):
        y = od.apply(x, int(g["drop_seed"]), call[0], float(g["drop_rate"]))
        call[0] += 1
        return y
    return drop


CALLS = [("c0", False, "small"), ("c1", True, "small"), ("bias", False, "small"), ("big", True, "big")]


@pytest.mark.parametrize("tag,concat,size", CALLS)
def test_oracle_and_the_aggregator_match_the_reference_class(golden, cpu_kernels, tag, concat, size):  # noqa: F811
    from oracle import pool2_forward as p2
    g, w = golden, _w(golden, tag + "_")
    want = g[tag + "_out"]
    assert np.allclose(p2.aggregator(g["self"], g["neigh"], w, concat), want, rtol=1e-5, atol=1e-6)
    a = gs.TwoMaxLayerPoolingAggregator(10, 6, model_size=size, bias="bias" in w, concat=concat, device="cpu")
    a.math = ops.MATH_FP32_SIMT
    assert [tuple(x.shape) for x in (a.mlp_layers[0].vars["weights"], a.mlp_layers[1].vars["weights"],
                                     a.vars["neigh_weights"], a.vars["self_weights"])] == [tuple(r[1:]) for r in
                                                                                          g[tag + "_draws"]]
    for layer, i in zip(a.mlp_layers, (1, 2)):
        layer.vars["weights"], layer.vars["bias"] = torch.from_numpy(w["W%d" % i]), torch.from_numpy(w["b%d" % i])
    for name in ("neigh_weights", "self_weights") + (("bias",) if "bias" in w else ()):
        a.vars[name] = torch.from_numpy(w[name])
    got = a((torch.from_numpy(g["self"]), torch.from_numpy(g["neigh"])))
    assert np.allclose(got.numpy(), want, rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize("tag", ["khop", "drop"])
def test_sample_aggregate_and_dropout_match_the_reference(golden, cpu_kernels, tag):  # noqa: F811
    """The reference's two-layer aggregate (concat, node 3's neighbours all the dummy id): the oracle, and the product's
    training branch (_PoolAggregateRowsFn, both layers) on the reference's samples; with dropout 0.5 the masks are the
    oracle's, drawn in the product's site order, which must be the reference's call order and element layout."""
    from oracle import pool2_forward as p2
    g = golden
    fan, dims, B = [int(x) for x in g["khop_fanout"]], [int(x) for x in g["khop_dims"]], len(g["khop_seeds"])
    support = [int(x) for x in g[tag + "_support"]]
    samples = [g["%s_samples%d" % (tag, h)] for h in range(len(fan) + 1)]
    ws = [_w(g, "%s_L%d_" % (tag, li)) for li in range(len(fan))]
    rate = float(g["drop_rate"]) if tag == "drop" else 0.0
    ref = p2.aggregate_khop(samples, g["khop_feats"], fan, support, B, ws, True, _counter_drop(g) if rate else None)
    assert np.allclose(ref, g[tag + "_out"], rtol=1e-5, atol=1e-6)
    L = len(fan)
    plan = sm.dropout_site_plan("twomaxpool", L)
    if rate:                                         # the reference's calls: [n*k, d_in] then [n*k, h1] per (layer, hop)
        shapes = []
        for layer, hop, role in plan:
            rows = B * support[hop] * fan[L - hop - 1]
            shapes.append((rows, (1 if layer == 0 else 2) * dims[layer] if role == "mlp" else 512, -1))
        assert [tuple(c) for c in g["drop_calls"]] == shapes
    # the product's branch on the same samples and weights
    src = torch.from_numpy(g["khop_feats"])
    counts = [B * s for s in support]
    seed = int(g["drop_seed"])
    call = {site: i for i, site in enumerate(plan)}
    for layer in range(L):
        a = gs.TwoMaxLayerPoolingAggregator((1 if layer == 0 else 2) * dims[layer], dims[layer + 1],
                                            act=gs.relu if layer < L - 1 else gs.identity, concat=True, device="cpu")
        a.math = ops.MATH_FP32_SIMT
        w = ws[layer]
        for dense, i in zip(a.mlp_layers, (1, 2)):
            dense.vars["weights"], dense.vars["bias"] = torch.from_numpy(w["W%d" % i]), torch.from_numpy(w["b%d" % i])
        a.vars["neigh_weights"], a.vars["self_weights"] = torch.from_numpy(w["neigh_weights"]), torch.from_numpy(w["self_weights"])
        sites = None
        if rate:
            sites = [tuple((seed, call[(layer, h, role)], rate) for role in ("mlp", "mlp2")) for h in range(L - layer)]
        segs = gs.models.layer_segments([torch.from_numpy(s) for s in samples], counts, fan, layer)
        src = sm._PoolAggregateRowsFn.apply(a, src, segs, *sm.layer_params(a), None, sites)
    assert np.allclose(src[:B].detach().numpy(), g[tag + "_out"], rtol=1e-5, atol=1e-5)
