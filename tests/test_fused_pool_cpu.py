"""CPU: the fused bf16 pooling-branch training path (fused_pool=True) - its refusals, that the default builds what it
built before, the B1 contract of oracle/pool_grad.py against fp64 autograd, and the autograd wiring of
_FusedPoolAggregateRowsFn with torch stand-ins for the kernels (TEST mocks only; the product has no such path)."""
import numpy as np
import pytest
import torch

import graphsage_b200 as gs
from graphsage_b200 import ops, supervised_models as sm
from oracle import pool_grad


class _Sampler(object):
    counter, counter_dev = 0, None


def _model(cls=gs.SupervisedGraphsage, agg="maxpool", k=(4, 3), F=10, features=None, **kw):
    N = 30
    feats = torch.randn(N + 1, F) if features is None else features
    adj = torch.zeros((N + 1, 8), dtype=torch.int32)
    infos = [gs.SAGEInfo("node", _Sampler(), k[0], 8), gs.SAGEInfo("node", _Sampler(), k[1], 8)]
    placeholders = dict({"batch_size": 4, "dropout": 0.}, **kw.pop("placeholders", {}))
    if cls is gs.SupervisedGraphsage:
        return cls(3, placeholders, feats, adj, np.ones(N), infos, aggregator_type=agg, device="cpu", **kw)
    return cls(placeholders, feats, adj, np.ones(N), infos, aggregator_type=agg, device="cpu", **kw)


@pytest.mark.parametrize("cls", [gs.SupervisedGraphsage, gs.UnsupervisedGraphsage])
def test_refusals_name_the_limit(cls):
    with pytest.raises(NotImplementedError, match="fanouts <= 128"):
        _model(cls, k=(129, 3), fused_pool=True)
    with pytest.raises(NotImplementedError, match="input widths <= 640"):
        _model(cls, F=641, fused_pool=True)
    with pytest.raises(NotImplementedError, match="dropout"):
        _model(cls, placeholders={"dropout": 0.5}, fused_pool=True)
    with pytest.raises(NotImplementedError, match="maxpool and meanpool"):
        _model(cls, agg="mean", fused_pool=True)
    for agg in ("maxpool", "meanpool"):
        assert _model(cls, agg=agg, fused_pool=True).fused_pool


def test_refusals_of_a_sharded_table_hidden_width_and_dropout_at_the_step():
    m = _model(fused_pool=True)
    m.features = type("Sharded", (), {"c_table": None, "shape": (31, 10)})()
    with pytest.raises(NotImplementedError, match="ShardedFeatures"):
        sm.refuse_fused_pool(m)
    m = _model(fused_pool=True)
    m.aggregators[1].hidden_dim = 200
    with pytest.raises(NotImplementedError, match="multiple of 128"):
        sm.refuse_fused_pool(m)
    with pytest.raises(NotImplementedError, match="dropout"):
        sm.differentiable_outputs(_model(fused_pool=True), torch.zeros(4, dtype=torch.int32), dropout=0.5)
    agg = _model(fused_pool=True).aggregators[0]
    segs = [ops.Seg(2, 129, neigh_ids=torch.zeros(2 * 129, dtype=torch.int32), self_ids=torch.zeros(2, dtype=torch.int32))]
    mv = agg.mlp_layers[0].vars
    with pytest.raises(NotImplementedError, match="fanout <= 128"):
        sm._FusedPoolAggregateRowsFn.apply(agg, torch.zeros(31, 10), segs, agg.vars["self_weights"],
                                           agg.vars["neigh_weights"], mv["weights"], mv["bias"], None, True)


@pytest.mark.parametrize("fused", [False, True])
def test_default_builds_what_it_built_before(monkeypatch, fused):
    a, b = _model(), _model(fused_pool=fused)
    assert a.fused_pool is False and b.fused_pool is fused
    assert [tuple(p.shape) for p in a.parameters()] == [tuple(p.shape) for p in b.parameters()]
    assert [type(x) for x in a.aggregators] == [type(x) for x in b.aggregators]
    assert type(b.optimizer) is torch.optim.Adam and not b.optimizer.param_groups[0]["capturable"]
    # the training pass picks the materialised Function by default, the fused one with fused_pool=True
    used = []
    for fn in (sm._PoolAggregateRowsFn, sm._FusedPoolAggregateRowsFn):
        monkeypatch.setattr(fn, "apply", staticmethod(lambda agg, src, *a, _fn=fn: used.append(_fn) or torch.zeros(
            (src.shape[0], 2 * agg.output_dim))))
    B = 4
    monkeypatch.setattr(b, "sample", lambda batch, infos, batch_size=None: (
        [torch.zeros(B * n, dtype=torch.int32) for n in (1, 3, 12)], [1, 3, 12]))
    sm.differentiable_outputs(b, torch.zeros(B, dtype=torch.int32))
    assert used == [sm._FusedPoolAggregateRowsFn if fused else sm._PoolAggregateRowsFn] * 2


def _grid(r, shape, lim=8.0):
    """multiples of 2^-4 in [-lim, lim]: exact in bf16, and fp32 sums of their products are exact"""
    return (r.randint(-int(lim * 16), int(lim * 16) + 1, size=shape) / 16.0).astype(np.float32)


@pytest.mark.parametrize("pool", ["max", "mean"])
def test_oracle_matches_fp64_autograd_with_exact_ties(pool):
    r = np.random.RandomState(1)
    n, k, K, hid = 9, 5, 7, 6
    X = _grid(r, (n * k, K), 2.0)
    X[0:k] = X[0]                                        # a whole group of identical rows: k-way ties
    X[k:k + 2] = X[k + 2]                                # a three-way tie
    W, b = _grid(r, (K, hid), 1.0), _grid(r, (hid,), 1.0)
    b[2] = -1000.0                                       # a column that is negative everywhere: hp = 0
    dhp = _grid(r, (n, hid), 4.0)
    Xt, Wt, bt = (torch.from_numpy(v).double().requires_grad_(True) for v in (X, W, b))
    pre = Xt @ Wt
    pre.retain_grad()
    h = torch.relu(pre + bt).reshape(n, k, hid)
    hp = h.amax(dim=1) if pool == "max" else h.mean(dim=1)
    (hp * torch.from_numpy(dhp).double()).sum().backward()
    got = pool_grad.dpre((X.astype(np.float64) @ W.astype(np.float64)).astype(np.float32), b, dhp, k, pool)
    assert np.allclose(got, pre.grad.numpy(), rtol=1e-6, atol=0)
    assert (got[:, 2] == 0).all()
    if pool == "max":
        assert (np.abs(got[:k]) > 0).sum() >= k          # the tied group shares its gradient
    parts = pool_grad.dbm_partials(got, n, k)
    assert np.allclose(pool_grad.dbm_combine(parts), bt.grad.numpy(), rtol=1e-6, atol=1e-6)


def test_bf16_round_is_nearest_even():
    x = np.array([1.0, 1.0 + 2 ** -8, 1.0 + 3 * 2 ** -8, -2.5, 1.0 + 2 ** -7], np.float32)
    assert pool_grad.bf16_round(x).tolist() == torch.from_numpy(x).bfloat16().float().tolist()


# ---- the autograd wiring with torch stand-ins for the kernels

def _fake_bf16_table(self, src, persistent):
    return src.detach().bfloat16()


def _fake_k4(table, n_groups, k, W, bias, packed, row_ids=None, row0=0, K=None, out=None, pool="max"):
    X = table[row_ids.long()].float() if row_ids is not None else table[row0:row0 + n_groups * k].float()
    h = torch.relu(X @ W.bfloat16().float() + bias).reshape(n_groups, k, -1)
    out.copy_(h.amax(dim=1) if pool == "max" else h.mean(dim=1))
    return out


def _fake_dp(table, n_groups, k, W, bias, packed, dhp, row_ids=None, row0=0, K=None, pool="max"):
    X = table[row_ids.long()].float() if row_ids is not None else table[row0:row0 + n_groups * k].float()
    pre = (X.double() @ W.bfloat16().double()).float()
    d = pool_grad.dpre(pre.numpy(), bias.detach().numpy(), dhp.detach().numpy(), k, pool)
    return {"X": X, "dpre": torch.from_numpy(d), "dP": torch.from_numpy(pool_grad.bf16_round(d)), "n": n_groups, "k": k}


def _fake_dw(table, n_groups, k, grad, dWm, dbm, row_ids=None, row0=0, K=None):
    dWm += grad["X"].t() @ grad["dP"]
    dbm += torch.from_numpy(pool_grad.dbm_combine(pool_grad.dbm_partials(grad["dpre"].numpy(), n_groups, k)))


def _fake_dx(grad, n_groups, k, W, packed_dx, out=None):
    return (grad["dP"] @ W.bfloat16().float().t())[:, :packed_dx.cols]


def _fake_gather_rows_f32(feats, ids=None, row0=0, n=None, out=None):
    r = feats[ids.long()] if ids is not None else feats[row0:row0 + n]
    out.copy_(r.float())
    return out


def _fake_sage_gemm(parts, combine=ops.COMBINE_ADD, bias=None, act=ops.ACT_NONE, math=None, out=None, packed=None):
    ys = [a[:, :k] @ w for (a, k, w) in parts]
    y = torch.cat(ys, dim=1) if combine == ops.COMBINE_CONCAT else sum(ys[1:], ys[0])
    return torch.relu(y) if act == ops.ACT_RELU else y


@pytest.fixture()
def cpu_kernels(monkeypatch):
    monkeypatch.setattr(gs.MaxPoolingAggregator, "_bf16_table", _fake_bf16_table)
    monkeypatch.setattr(ops, "maxpool_mlp_fused", _fake_k4)
    monkeypatch.setattr(ops, "pool_mlp_backward_dp", _fake_dp)
    monkeypatch.setattr(ops, "pool_mlp_backward_dw", _fake_dw)
    monkeypatch.setattr(ops, "pool_mlp_backward_dx", _fake_dx)
    monkeypatch.setattr(ops, "gather_rows_f32", _fake_gather_rows_f32)
    monkeypatch.setattr(ops, "sage_gemm", _fake_sage_gemm)
    monkeypatch.setattr(ops, "PackedMlpWeights", lambda: None)
    monkeypatch.setattr(ops, "PackedMlpDxWeights", lambda cols: type("P", (), {"cols": cols})())


def _bf16_value(x):
    """x rounded to bf16 in the forward, identity in the backward (the kernels read bf16 operands, the gradient is fp32)"""
    return x + (x.detach().bfloat16().float() - x.detach())


def _ref_layer(selfv, neigh, k, w, pool, concat, last):
    n = selfv.shape[0]
    h = torch.relu(_bf16_value(neigh) @ _bf16_value(w["mlp_weights"]) + w["mlp_bias"]).reshape(n, k, -1)
    hp = h.amax(dim=1) if pool == "max" else h.mean(dim=1)
    fs, fn = selfv @ w["self_weights"], hp @ w["neigh_weights"]
    y = torch.cat([fs, fn], dim=1) if concat else fs + fn
    return y if last else torch.relu(y)


@pytest.mark.parametrize("pool", ["max", "mean"])
@pytest.mark.parametrize("concat", [True, False])
def test_fused_function_wiring_matches_autograd(cpu_kernels, pool, concat):
    r = np.random.RandomState(3)
    N, F, D, B, k1, k2 = 40, 10, 6, 5, 3, 4
    feats = torch.from_numpy(_grid(r, (N, F), 1.0))
    s0 = torch.from_numpy(r.randint(0, N, size=B).astype(np.int32))
    s1 = torch.from_numpy(r.randint(0, N, size=B * k1).astype(np.int32))
    s2 = torch.from_numpy(r.randint(0, N, size=B * k1 * k2).astype(np.int32))
    cls = gs.MaxPoolingAggregator if pool == "max" else gs.MeanPoolingAggregator
    dm = 2 if concat else 1
    a0 = cls(F, D, act=gs.relu, concat=concat, device="cpu")
    a1 = cls(dm * D, D, act=gs.identity, concat=concat, device="cpu")
    params = []
    for a in (a0, a1):
        a.mlp_layers[0].vars["bias"] = torch.from_numpy(r.randn(a.hidden_dim).astype(np.float32) * 0.1)
        for d in (a.vars, a.mlp_layers[0].vars):
            for key in d:
                d[key] = d[key].detach().clone().requires_grad_(True)
                params.append(d[key])
    seg0 = [ops.Seg(B, k1, self_ids=s0, neigh_ids=s1, out_row0=0), ops.Seg(B * k1, k2, self_ids=s1, neigh_ids=s2, out_row0=B)]
    m0, m1 = a0.mlp_layers[0].vars, a1.mlp_layers[0].vars
    h1 = sm._FusedPoolAggregateRowsFn.apply(a0, feats, seg0, a0.vars["self_weights"], a0.vars["neigh_weights"],
                                            m0["weights"], m0["bias"], None, True)
    seg1 = [ops.Seg(B, k1, self_row0=0, neigh_row0=B, out_row0=0)]
    out = sm._FusedPoolAggregateRowsFn.apply(a1, h1, seg1, a1.vars["self_weights"], a1.vars["neigh_weights"],
                                             m1["weights"], m1["bias"], None, False)
    R = torch.from_numpy(r.randn(*out.shape).astype(np.float32))
    (out * R).sum().backward()
    got = [p.grad.clone() for p in params]
    for p in params:
        p.grad = None
    w0 = dict(a0.vars, mlp_weights=m0["weights"], mlp_bias=m0["bias"])
    w1 = dict(a1.vars, mlp_weights=m1["weights"], mlp_bias=m1["bias"])
    x0, x1, x2 = feats[s0.long()], feats[s1.long()], feats[s2.long()]
    ref = _ref_layer(_ref_layer(x0, x1, k1, w0, pool, concat, False), _ref_layer(x1, x2, k2, w0, pool, concat, False),
                     k1, w1, pool, concat, True)
    assert torch.allclose(out.detach(), ref.detach(), rtol=1e-2, atol=1e-2)
    (ref * R).sum().backward()
    for p, g in zip(params, got):
        assert p.grad is not None
        err = float((g - p.grad).norm() / max(float(p.grad.norm()), 1e-12))
        assert err < 2e-2, err
