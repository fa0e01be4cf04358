"""Training dropout without a GPU: the Philox mask contract (oracle/dropout.py), the reference's dropout call order pinned by
tests/golden/dropout.npz, and the autograd wiring of the dropout paths (_AggregateRowsFn, _PoolAggregateRowsFn, the head)
with the kernels replaced by torch stand-ins that draw the oracle's masks - TEST mocks only, the product has no such path.
The GPU twin (test_zz_gpu_dropout.py) drives the real kernels."""
import os

import numpy as np
import pytest
import torch

import graphsage_b200 as gs
from graphsage_b200 import ops, supervised_models as sm
from oracle import dropout as od
from oracle.aggregate import l2_normalize

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "dropout.npz")


# ---------------------------------------------------------------------------------------------------- mask contract
@pytest.mark.parametrize("rate", [0.1, 0.5, 0.9])
def test_keep_rate_within_five_sigma(rate):
    m = od.keep_mask(77, 3, rate, np.arange(1000), 1000)
    q = 1.0 - rate
    n = m.size
    assert abs(m.sum() - n * q) < 5 * np.sqrt(n * q * (1 - q))


def test_masks_of_different_calls_positions_and_column_groups_are_uncorrelated():
    rate, n = 0.5, 200000
    a = od.keep_mask(5, 0, rate, np.arange(n), 4).astype(np.float64)
    b = od.keep_mask(5, 1, rate, np.arange(n), 4).astype(np.float64)         # another call
    c = od.keep_mask(5, 0, rate, np.arange(n) + n, 4).astype(np.float64)     # other positions
    d = od.keep_mask(5, 0, rate, np.arange(n), 8)[:, 4:].astype(np.float64)  # the next column group
    e = od.keep_mask(6, 0, rate, np.arange(n), 4).astype(np.float64)         # another seed
    bound = 5.0 / np.sqrt(a.size)
    for other in (b, c, d, e):
        assert abs(np.corrcoef(a.ravel(), other.ravel())[0, 1]) < bound
    for i in range(4):                                                      # the four words of one block
        for j in range(i + 1, 4):
            assert abs(np.corrcoef(a[:, i], a[:, j])[0, 1]) < 5.0 / np.sqrt(n)


def test_rate_zero_is_the_identity_and_bad_rates_are_refused():
    x = np.random.RandomState(0).randn(37, 13).astype(np.float32)
    assert np.array_equal(od.apply(x, 9, 4, 0.0), x)
    for bad in (-0.1, 1.0, 1.5):
        with pytest.raises(ValueError):
            od.threshold(bad)
        with pytest.raises(ValueError):
            ops.dropout_site((1, 2, bad))


def test_kept_elements_are_divided_by_fp32_keep():
    x = np.full((64, 9), 3.0, np.float32)
    y = od.apply(x, 1, 2, 0.3)
    keep = np.float32(1.0 - np.float64(np.float32(0.3)))
    assert set(np.unique(y)) <= {np.float32(0), np.float32(3.0) / keep}


# ---------------------------------------------------------------------------------------------------- reference call order
def _cases():
    return [("mean", False), ("mean", True), ("gcn", False), ("maxpool", False), ("maxpool", True), ("meanpool", False),
            ("meanpool", True)]


def _weights(g, key, L):
    out = []
    for li in range(L):
        w = {}
        for name in ("self_weights", "neigh_weights", "weights", "mlp_weights", "mlp_bias"):
            if "%sL%d_%s" % (key, li, name) in g:
                w[name] = g["%sL%d_%s" % (key, li, name)]
        out.append(w)
    return out


def _plan_shapes(kind, fan, dims, concat, B, head):
    """The shape of every site's tensor, in the product's site order (supervised_models.dropout_site_plan)."""
    L = len(fan)
    support = [int(np.prod(fan[L - h:])) if h else 1 for h in range(L + 1)]
    shapes = []
    for layer, hop, role in sm.dropout_site_plan(kind, L, head=head):
        if role == "head":
            shapes.append((B, (2 if concat else 1) * dims[-1], -1))
            continue
        n, k = B * support[hop], fan[L - hop - 1]
        F = (2 if concat and layer else 1) * dims[layer]
        shapes.append({"neigh": (n, k, F), "self": (n, F, -1), "mlp": (n * k, F, -1)}[role])
    return np.array(shapes, dtype=np.int64)


@pytest.mark.parametrize("kind,concat", _cases())
def test_oracle_restates_the_reference_with_dropout_and_the_site_order_matches(kind, concat):
    g = np.load(GOLDEN)
    key = "%s_c%d_" % (kind, int(concat))
    fan, dims, rate, seed = [int(x) for x in g["fanout"]], [int(x) for x in g["dims"]], float(g["rate"]), int(g["seed"])
    L = len(fan)
    support = [1, fan[1], fan[1] * fan[0]]
    w = _weights(g, key, L)
    # supervised: the aggregate pass, then the head's site
    B = len(g["seeds"])
    samples = [g["%ssup_samples%d" % (key, h)] for h in range(L + 1)]
    out, call = od.aggregate_khop(samples, g["feats"], fan, support, B, w, concat, kind, rate, seed, 0)
    assert np.abs(out - g[key + "sup_out"]).max() < 1e-5
    logits = od.apply(l2_normalize(out), seed, call, rate) @ g[key + "head_w"] + g[key + "head_b"]
    assert np.abs(logits - g[key + "sup_logits"]).max() < 1e-5
    assert np.array_equal(g[key + "sup_calls"], _plan_shapes(kind, fan, dims, concat, B, head=True))
    # unsupervised: batch1, batch2, negatives - each pass numbers its sites after the previous pass's
    call, shapes = 0, []
    for tag, bs in (("u1", B), ("u2", B), ("un", len(g["neg"]))):
        samples = [g["%s%s_samples%d" % (key, tag, h)] for h in range(L + 1)]
        out, call = od.aggregate_khop(samples, g["feats"], fan, support, bs, w, concat, kind, rate, seed, call)
        assert np.abs(out - g[key + tag + "_out"]).max() < 1e-5
        shapes.append(_plan_shapes(kind, fan, dims, concat, bs, head=False))
    assert np.array_equal(g[key + "unsup_calls"], np.concatenate(shapes))


# ---------------------------------------------------------------------------------------------------- autograd wiring
def _mask(site, rows, F):
    seed, call, rate = site
    return torch.from_numpy(od.keep_mask(seed, call, rate, np.arange(rows), F))


def _keep(site):
    return float(od.keep_prob(site[2]))


def _fake_dropout_apply(x, site, rows=None, group=1, scale=1.0, out=None, accumulate=False):
    rows = x.shape[0] * group if rows is None else rows
    xr = x.repeat_interleave(group, dim=0)[:rows]
    v = torch.where(_mask(site, rows, x.shape[1]), (xr * scale) / _keep(site), torch.zeros((), dtype=x.dtype))
    if out is None:
        return v
    if accumulate:
        out[:rows] += v
    else:
        out[:rows] = v
    return out


def _rows(src, ids, row0, n):
    return src[ids[:n].long()] if ids is not None else src[row0:row0 + n]


def _fake_gather_mean_dropout(src, segments, neigh_sites, self_sites, include_self=False, want_self=True, out_pitch=None):
    rows, F = max(s.out_row0 + s.n for s in segments), src.shape[1]
    xs, xm = torch.zeros(rows, F), torch.zeros(rows, F)
    for s, ns, ss in zip(segments, neigh_sites, self_sites):
        nb = _fake_dropout_apply(_rows(src, s.neigh_ids, s.neigh_row0, s.n * s.k), ns).reshape(s.n, s.k, F)
        sv = _fake_dropout_apply(_rows(src, s.self_ids, s.self_row0, s.n), ss)
        allv = torch.cat([nb, sv[:, None]], dim=1) if include_self else nb
        xm[s.out_row0:s.out_row0 + s.n] = allv.mean(dim=1)
        xs[s.out_row0:s.out_row0 + s.n] = sv
    return (xs if want_self else None), xm


def _fake_embedding_grad(lists, n_rows, d, out=None, sites=None):
    out = torch.zeros(n_rows, d)
    for li, (ids, grad, group, scale) in enumerate(lists):
        n = ids.numel()
        g = grad[:, :d].repeat_interleave(group, dim=0)[:n] * scale
        if sites is not None:
            g = torch.where(_mask(sites[li], n, d), g / _keep(sites[li]), torch.zeros(()))
        out.index_add_(0, ids.long(), g)
    return out


def _fake_sage_gemm(parts, combine=ops.COMBINE_ADD, bias=None, act=ops.ACT_NONE, math=None, out=None, packed=None):
    ys = [a[:, :k] @ w for (a, k, w) in parts]
    y = torch.cat(ys, dim=1) if combine == ops.COMBINE_CONCAT else sum(ys[1:], ys[0])
    if bias is not None:
        y = y + bias
    return torch.relu(y) if act == ops.ACT_RELU else y


def _fake_gather_rows(feats, ids, out=None):
    r = feats[ids.long()].float()
    if out is not None:
        out.copy_(r)
        return out
    return r


def _fake_gather_mean(src, segments, include_self=False, want_self=True, out_pitch=None, out_mean=None, out_self=None):
    (s,) = segments
    return None, src[s.neigh_row0:s.neigh_row0 + s.n * s.k].reshape(s.n, s.k, -1).mean(dim=1)


@pytest.fixture()
def cpu_kernels(monkeypatch):
    monkeypatch.setattr(ops, "sage_gemm", _fake_sage_gemm)
    monkeypatch.setattr(ops, "gather_rows", _fake_gather_rows)
    monkeypatch.setattr(ops, "gather_mean", _fake_gather_mean)
    monkeypatch.setattr(ops, "segment_max", lambda x, n, k: x.reshape(n, k, -1).amax(dim=1))
    monkeypatch.setattr(ops, "gather_mean_dropout", _fake_gather_mean_dropout)
    monkeypatch.setattr(ops, "dropout_apply", _fake_dropout_apply)
    monkeypatch.setattr(ops, "embedding_grad", _fake_embedding_grad)


def _tdrop(x, site):
    """drop(x) as differentiable torch: x / keep * mask."""
    return x / _keep(site) * _mask(site, x.shape[0], x.shape[1]).to(x.dtype)


def _ref_layer(kind, selfv, neigh, k, w, sites, concat, last):
    """The oracle's op sequence with dropout in differentiable torch.  neigh: [n * k, F] rows."""
    n, F = selfv.shape
    if kind in ("mean", "gcn"):
        nb = _tdrop(neigh, sites[0]).reshape(n, k, F)
        sv = _tdrop(selfv, sites[1])
        if kind == "gcn":
            y = torch.cat([nb, sv[:, None]], dim=1).mean(dim=1) @ w["weights"]
            return y if last else torch.relu(y)
        fs, fn = sv @ w["self_weights"], nb.mean(dim=1) @ w["neigh_weights"]
    else:
        h = torch.relu(_tdrop(neigh, sites) @ w["mlp_weights"] + w["mlp_bias"]).reshape(n, k, -1)
        hp = h.amax(dim=1) if kind == "maxpool" else h.mean(dim=1)
        fs, fn = selfv @ w["self_weights"], hp @ w["neigh_weights"]
    y = torch.cat([fs, fn], dim=1) if concat else fs + fn
    return y if last else torch.relu(y)


@pytest.mark.parametrize("kind,concat", _cases())
@pytest.mark.parametrize("rate", [0.1, 0.5])
def test_two_layer_dropout_chain_gradients_match_autograd(cpu_kernels, kind, concat, rate):
    r = np.random.RandomState(11)
    N, F, d, D, B, k1, k2 = 40, 10, 3, 6, 5, 3, 4
    feats = torch.from_numpy(r.randn(N, F).astype(np.float32))
    emb = torch.from_numpy(r.randn(N, d).astype(np.float32)).requires_grad_(True)
    table = torch.cat([emb.detach(), feats], dim=1)                  # embeddings first, as the product's table
    s0 = torch.from_numpy(r.randint(0, N, size=B).astype(np.int32))
    s1 = torch.from_numpy(r.randint(0, N, size=B * k1).astype(np.int32))
    s2 = torch.from_numpy(r.randint(0, N, size=B * k1 * k2).astype(np.int32))
    s2[:5] = 7                                                        # repeated ids: several contributions per row
    cls = {"mean": gs.MeanAggregator, "gcn": gs.GCNAggregator, "maxpool": gs.MaxPoolingAggregator,
           "meanpool": gs.MeanPoolingAggregator}[kind]
    pool = kind in ("maxpool", "meanpool")
    dim_mult = 2 if concat else 1
    a0 = cls(F + d, D, act=gs.relu, concat=concat, device="cpu")
    a1 = cls(dim_mult * D, D, act=gs.identity, concat=concat, device="cpu")
    params = []
    for a in (a0, a1):
        a.math = ops.MATH_FP32_SIMT
        dicts = [a.vars] + ([a.mlp_layers[0].vars] if pool else [])
        if pool:
            a.mlp_layers[0].vars["bias"] = torch.from_numpy(r.randn(a.hidden_dim).astype(np.float32) * 0.1)
        for dct in dicts:
            for key in dct:
                dct[key] = dct[key].detach().clone().requires_grad_(True)
                params.append(dct[key])
    seed = 99
    if pool:
        sites0 = [(seed, 0, rate), (seed, 1, rate)]
        sites1 = [(seed, 2, rate)]
    else:
        sites0 = [((seed, 0, rate), (seed, 1, rate)), ((seed, 2, rate), (seed, 3, rate))]
        sites1 = [((seed, 4, rate), (seed, 5, rate))]

    def apply(a, src, segs, e, sites):
        if pool:
            m = a.mlp_layers[0].vars
            return sm._PoolAggregateRowsFn.apply(a, src, segs, a.vars["self_weights"], a.vars["neigh_weights"], m["weights"],
                                                 m["bias"], e, sites)
        ws = (a.vars["weights"],) if kind == "gcn" else (a.vars["self_weights"], a.vars["neigh_weights"])
        return sm._AggregateRowsFn.apply(a, src, segs, e, sites, *ws)

    seg0 = [ops.Seg(B, k1, self_ids=s0, neigh_ids=s1, out_row0=0), ops.Seg(B * k1, k2, self_ids=s1, neigh_ids=s2, out_row0=B)]
    h1 = apply(a0, table, seg0, emb, sites0)
    out = apply(a1, h1, [ops.Seg(B, k1, self_row0=0, neigh_row0=B, out_row0=0)], None, sites1)
    R = torch.from_numpy(r.randn(*out.shape).astype(np.float32))
    (out * R).sum().backward()
    got = [p.grad.clone() for p in params] + [emb.grad.clone()]
    for p in params + [emb]:
        p.grad = None

    def wd(a):
        w = dict(a.vars)
        if pool:
            w.update(mlp_weights=a.mlp_layers[0].vars["weights"], mlp_bias=a.mlp_layers[0].vars["bias"])
        return w

    full = torch.cat([emb, feats], dim=1)
    x0, x1, x2 = full[s0.long()], full[s1.long()], full[s2.long()]
    r0 = _ref_layer(kind, x0, x1, k1, wd(a0), sites0[0], concat, last=False)
    r1 = _ref_layer(kind, x1, x2, k2, wd(a0), sites0[1], concat, last=False)
    ref = _ref_layer(kind, r0, r1, k1, wd(a1), sites1[0], concat, last=True)
    assert torch.allclose(out.detach(), ref.detach(), rtol=1e-5, atol=1e-5)
    (ref * R).sum().backward()
    for p, g in zip(params + [emb], got):
        assert p.grad is not None and torch.allclose(g, p.grad, rtol=2e-4, atol=2e-5), float((g - p.grad).abs().max())


def test_head_dropout_backward_applies_the_same_mask(cpu_kernels):
    x = torch.randn(9, 7, requires_grad=True)
    site = (3, 17, 0.5)
    y = sm._DropoutFn.apply(x, site)
    R = torch.randn(9, 7)
    (y * R).sum().backward()
    x2 = x.detach().clone().requires_grad_(True)
    ref = _tdrop(x2, site)
    (ref * R).sum().backward()
    assert torch.allclose(y, ref) and torch.allclose(x.grad, x2.grad)


def test_site_plan_follows_the_reference_call_order():
    assert sm.dropout_site_plan("mean", 2, head=True) == [(0, 0, "neigh"), (0, 0, "self"), (0, 1, "neigh"), (0, 1, "self"),
                                                           (1, 0, "neigh"), (1, 0, "self"), (None, None, "head")]
    assert sm.dropout_site_plan("maxpool", 2) == [(0, 0, "mlp"), (0, 1, "mlp"), (1, 0, "mlp")]
