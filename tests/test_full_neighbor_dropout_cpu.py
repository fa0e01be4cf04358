"""CPU: full-neighbourhood training with dropout.  The oracle (oracle/full_neighbor_dropout.py) against a dense
restatement and float64 autograd, its minibatch blocks against its whole-graph pass bit for bit, the site plan, the
`dropout=` argument's semantics and refusals, and the model's autograd wiring with the oracle standing in for the kernels."""
import numpy as np
import pytest
import torch

import graphsage_b200 as gs
import oracle.full_neighbor_dropout as fd
from graphsage_b200 import full_neighbor_training as fnt
from graphsage_b200 import ops
from graphsage_b200.aggregators import MeanAggregator
from graphsage_b200.supervised_models import SupervisedGraphsage, full_neighbor_site_plan
from graphsage_b200.unsupervised_models import UnsupervisedGraphsage
from oracle.dropout import keep_mask, keep_prob


def messy_graph(N=24, seed=0):
    """Empty rows, duplicates, self loops, out-of-range entries (-1, N, N + 7) and one long row."""
    r = np.random.RandomState(seed)
    rows = []
    for i in range(N):
        k = 0 if i % 7 == 3 else int(r.randint(1, 5))
        e = list(r.randint(0, N, size=k))
        if i % 5 == 1 and e:
            e += [e[0], i]
        if i % 6 == 2:
            e += [-1, N, N + 7]
        rows.append(e)
    rows[N - 1] = list(r.randint(0, N, size=40))
    indptr = np.zeros(N + 1, np.int64)
    indptr[1:] = np.cumsum([len(x) for x in rows])
    return indptr, np.array([v for x in rows for v in x], np.int32)


SITE, SELF = (5, 11, 0.5), (5, 12, 0.3)


@pytest.mark.parametrize("op", ["mean", "mean_self"])
@pytest.mark.parametrize("rows", [None, [0, 3, 3, 23, 24, -2]])
def test_masked_forward_matches_the_dense_restatement(op, rows):
    indptr, indices = messy_graph()
    N = len(indptr) - 1
    x = np.random.RandomState(1).randn(N + 1, 7).astype(np.float32)
    rows_ = None if rows is None else np.array(rows)
    got = fd.csr_aggregate_dropout(x, indptr, indices, op, SITE, SELF, (indptr, None, len(indices)), rows_)
    ref = fd.dense_masked_mean(x, indptr, indices, op, SITE, SELF, rows_)
    assert np.abs(got - ref).max() <= 1e-5 * max(1, np.abs(ref).max())
    # rate 0 is the unmasked reduction, bit for bit
    import oracle.full_neighbor as fn
    z = fd.csr_aggregate_dropout(x, indptr, indices, op, (5, 11, 0.), (5, 12, 0.), (indptr, None, len(indices)), rows_)
    assert np.array_equal(z, fn.csr_aggregate(x, indptr, indices, op, rows_))


@pytest.mark.parametrize("with_self", [False, True])
def test_transpose_slots_name_every_forward_entry(with_self):
    indptr, indices = messy_graph(seed=2)
    N = len(indptr) - 1
    t_indptr, t_indices, t_slot = fd.csr_transpose_slots(indptr, indices, with_self)
    from oracle.full_neighbor_grad import csr_transpose
    a, b = csr_transpose(indptr, indices, with_self)
    assert np.array_equal(a, t_indptr) and np.array_equal(b, t_indices)
    for j in range(N + 1):
        for k in range(t_indptr[j], t_indptr[j + 1]):
            i, s = t_indices[k], t_slot[k]
            if s >= 0:
                e = indices[indptr[i] + s]
                assert (e if 0 <= e <= N else N) == j
            elif s == -1:
                assert j == N and (i == N or indptr[i + 1] <= indptr[i])
            else:
                assert with_self and s == -2 and i == j


def test_masked_sum_is_the_transpose_of_the_masked_mean():
    """<g, mean_drop(x)> = <mean_backward_drop(g), x>: the backward regenerates exactly the forward's masks."""
    indptr, indices = messy_graph(seed=4)
    N = len(indptr) - 1
    r = np.random.RandomState(2)
    x, g = r.randn(N + 1, 6).astype(np.float32), r.randn(N + 1, 6).astype(np.float32)
    pm = (indptr, None, len(indices))
    for with_self in (False, True):
        y = fd.csr_aggregate_dropout(x, indptr, indices, "mean_self" if with_self else "mean", SITE, SELF, pm)
        dx = fd.mean_backward_dropout(g, indptr, indices, with_self, SITE, SELF, pm)
        lhs, rhs = float((g.astype(np.float64) * y).sum()), float((dx.astype(np.float64) * x).sum())
        assert abs(lhs - rhs) <= 1e-4 * max(1.0, abs(lhs))


def _agg_dicts(kind, dims, concat, r):
    aggs = []
    for l in range(len(dims) - 1):
        din = dims[l] * (2 if concat and l and kind != "gcn" else 1)
        w = lambda *s: (r.randn(*s) * 0.5).astype(np.float32)          # noqa: E731
        if kind == "gcn":
            aggs.append(dict(type="gcn", weights=w(din, dims[l + 1])))
        elif kind == "mean":
            aggs.append(dict(type="mean", self_weights=w(din, dims[l + 1]), neigh_weights=w(din, dims[l + 1])))
        else:
            aggs.append(dict(type=kind, mlp_weights=w(din, 8), mlp_bias=w(8) * 0.1, self_weights=w(din, dims[l + 1]),
                             neigh_weights=w(8, dims[l + 1])))
    return aggs


@pytest.mark.parametrize("kind", ["mean", "gcn", "maxpool", "meanpool"])
@pytest.mark.parametrize("L", [1, 2, 3])
def test_blocks_mask_as_the_whole_graph_does(kind, L):
    indptr, indices = messy_graph(seed=7)
    N = len(indptr) - 1
    r = np.random.RandomState(3)
    feats = np.vstack([r.randn(N, 5).astype(np.float32), np.zeros((1, 5), np.float32)])
    concat = kind != "gcn"
    aggs = _agg_dicts(kind, [5] + [4] * L, concat, r)
    seeds = np.array([3, 0, 23, 23, 11, -4, N + 2])
    sites = fd.sites(kind, L, False, 99, 40, 0.4)
    whole = fd.full_neighbor_outputs(feats, indptr, indices, aggs, concat, seeds, sites)
    blocks = fd.block_outputs(feats, indptr, indices, aggs, concat, seeds, sites)
    assert np.array_equal(whole, blocks)
    other = fd.full_neighbor_outputs(feats, indptr, indices, aggs, concat, seeds, fd.sites(kind, L, False, 99, 41, 0.4))
    assert not np.array_equal(whole, other)


def _torch_formula(feats, indptr, indices, aggs, concat, node_ids, pw, pb, labels, sites, wd, d):
    """The masked loss in float64 torch from explicit per-entry and per-node mask tensors (amax splits ties evenly)."""
    N, nnz = len(indptr) - 1, len(indices)
    dst, src, pos = [], [], []
    for v in range(N + 1):
        c = indptr[v + 1] - indptr[v] if v < N else 0
        if c > 0:
            e = indices[indptr[v]:indptr[v + 1]].astype(np.int64)
            dst += [v] * c
            src += list(np.where((e < 0) | (e > N), N, e))
            pos += list(indptr[v] + np.arange(c))
        else:
            dst, src, pos = dst + [v], src + [N], pos + [nnz + v]
    dst, src, pos = (torch.tensor(np.array(a, np.int64)) for a in (dst, src, pos))
    cnt = torch.bincount(dst, minlength=N + 1).to(torch.float64).unsqueeze(1)

    def mask(site, p, F):
        return torch.from_numpy(keep_mask(*site, np.asarray(p), F).astype(np.float64)) / float(keep_prob(site[2]))

    emb = torch.from_numpy(feats[:, :d].astype(np.float64)).requires_grad_(True) if d else None
    h = torch.from_numpy(feats.astype(np.float64))
    if d:
        h = torch.cat([emb, h[:, d:]], dim=1)
    params = [{k: torch.from_numpy(v.astype(np.float64)).requires_grad_(True) for k, v in a.items() if k != "type"}
              for a in aggs]
    ids = torch.from_numpy(np.asarray(node_ids, np.int64))
    nodes = torch.arange(N + 1)
    for l, (a, p) in enumerate(zip(aggs, params)):
        last = l == len(aggs) - 1
        F = h.shape[1]
        if a["type"] in ("mean", "gcn"):
            msg = h[src] * mask(sites[(l, "neigh")], pos, F)
            s = torch.zeros_like(h).index_add(0, dst, msg)
            if a["type"] == "gcn":
                y = ((s + h * mask(sites[(l, "self")], nodes, F)) / (cnt + 1)) @ p["weights"]
            else:
                fs = (h * mask(sites[(l, "self")], nodes, F)) @ p["self_weights"]
                fn_ = (s / cnt) @ p["neigh_weights"]
                y = torch.cat([fs, fn_], 1) if concat else fs + fn_
        else:
            z = torch.relu((h * mask(sites[(l, "mlp")], nodes, F)) @ p["mlp_weights"] + p["mlp_bias"])
            if a["type"] == "maxpool":
                nb = torch.zeros_like(z[:, :]).scatter_reduce(0, dst.unsqueeze(1).expand(-1, z.shape[1]), z[src], "amax",
                                                                include_self=False)
            else:
                nb = torch.zeros_like(z).index_add(0, dst, z[src]) / cnt
            fs, fn_ = h @ p["self_weights"], nb @ p["neigh_weights"]
            y = torch.cat([fs, fn_], 1) if concat else fs + fn_
        h = y[ids] if last else torch.relu(y)
    out = h / torch.sqrt(torch.clamp((h * h).sum(1, keepdim=True), min=1e-12))
    out = out * mask(sites[(None, "head")], np.arange(len(node_ids)), out.shape[1])
    W = torch.from_numpy(pw.astype(np.float64)).requires_grad_(True)
    b = torch.from_numpy(pb.astype(np.float64)).requires_grad_(True)
    loss = (-(torch.from_numpy(labels) * torch.log_softmax(out @ W + b, 1)).sum(1)).mean()
    decayed = [W, b] + [v for p in params for k, v in p.items() if not k.startswith("mlp")]
    loss = loss + wd * 0.5 * sum((v * v).sum() for v in decayed)
    loss.backward()
    return float(loss.detach()), [{k: v.grad.numpy() for k, v in p.items()} for p in params], \
        {"weights": W.grad.numpy(), "bias": b.grad.numpy()}, (emb.grad.numpy() if d else None)


@pytest.mark.parametrize("kind", ["mean", "gcn", "maxpool", "meanpool"])
@pytest.mark.parametrize("concat", [True, False])
@pytest.mark.parametrize("d,L", [(0, 1), (16, 2), (0, 3)])
def test_oracle_backward_equals_float64_autograd(kind, concat, d, L):
    r = np.random.RandomState(8)
    indptr, indices = messy_graph(seed=9)
    N, F, C = len(indptr) - 1, 5, 3
    x = r.randint(0, 3, size=(N + 1, F)).astype(np.float32) if kind == "maxpool" else r.randn(N + 1, F).astype(np.float32)
    x[N] = 0
    feats = np.concatenate([r.randn(N + 1, d).astype(np.float32), x], 1) if d else x
    aggs = _agg_dicts(kind, [d + F] + [4] * L, concat, r)
    node_ids = np.array([0, 3, 5, 5, 9, 2, 11, 3, 23], np.int64)
    out_w = 4 * (2 if concat and kind != "gcn" else 1)
    pw, pb = (r.randn(out_w, C) * 0.5).astype(np.float32), (r.randn(C) * 0.1).astype(np.float32)
    labels = np.eye(C)[r.randint(0, C, len(node_ids))]
    sites = fd.sites(kind, L, True, 31, 7, 0.5)
    loss, grads, head, demb = fd.full_neighbor_loss_grads(feats, indptr, indices, aggs, concat, node_ids, labels, pw, pb,
                                                          sites, False, 0.01, d)
    rl, rg, rh, rd = _torch_formula(feats, indptr, indices, aggs, concat, node_ids, pw, pb, labels, sites, 0.01, d)
    assert abs(loss - rl) < 1e-5 * max(1, abs(rl))

    def close(a, b, what):
        assert np.abs(a - b).max() <= 1e-4 * max(1.0, np.abs(b).max()), (what, np.abs(a - b).max())
    for l, (g, ref) in enumerate(zip(grads, rg)):
        assert set(g) == set(ref)
        for k in g:
            close(g[k], ref[k], (l, k))
    close(head["weights"], rh["weights"], "head")
    if d:
        close(demb, rd, "embeddings")


def test_site_plan():
    assert full_neighbor_site_plan("mean", 2) == [(0, "neigh"), (0, "self"), (1, "neigh"), (1, "self")]
    assert full_neighbor_site_plan("gcn", 1, head=True) == [(0, "neigh"), (0, "self"), (None, "head")]
    assert full_neighbor_site_plan("maxpool", 3) == [(0, "mlp"), (1, "mlp"), (2, "mlp")]
    assert full_neighbor_site_plan("meanpool", 2, True) == [(0, "mlp"), (1, "mlp"), (None, "head")]
    assert [k for k in fd.sites("mean", 2, True, 1, 0, .5)] == full_neighbor_site_plan("mean", 2, True)


# ---------------------------------------------------------------- the argument and the refusals (they fire first)
CSR = (np.zeros(5, np.int64), np.zeros(0, np.int32))


def _bare_model(**attrs):
    m = SupervisedGraphsage.__new__(SupervisedGraphsage)
    m.aggregator_cls = MeanAggregator
    m.features = torch.zeros((5, 3))
    m.device = torch.device("cpu")
    m.aggregators = None
    m.distributed, m.dropout_rate = False, 0.
    for k, v in attrs.items():
        setattr(m, k, v)
    return m


@pytest.mark.parametrize("bad", [-0.1, 1.0, 1.5, float("nan"), "0.5", True, [0.5]])
def test_invalid_dropout_is_a_value_error(bad):
    for call in (lambda m: m.full_neighbor_train_step(*CSR, [0], [[1.0]], dropout=bad),
                 lambda m: m.full_neighbor_minibatch_loss(*CSR, [0], [[1.0]], dropout=bad),
                 lambda m: m.full_neighbor_outputs(*CSR, [0], dropout=bad)):
        with pytest.raises(ValueError, match="dropout"):
            call(_bare_model(dropout_rate=0.5))


def test_refusals_are_unchanged():
    with pytest.raises(NotImplementedError, match="dropout"):
        _bare_model(dropout_rate=0.5).full_neighbor_train_step(*CSR, [0], [[1.0]])
    with pytest.raises(NotImplementedError, match="dropout"):
        _bare_model(dropout_rate=0.5).full_neighbor_minibatch_outputs(*CSR, [0], dropout=None)
    with pytest.raises(NotImplementedError, match="distributed"):
        _bare_model(distributed=True).full_neighbor_loss(*CSR, [0], [[1.0]], dropout=0.5)
    m = _bare_model()
    m.features = type("Sharded", (), {"c_table": lambda self: None, "shape": (5, 3)})()
    with pytest.raises(NotImplementedError, match="ShardedFeatures"):
        m.full_neighbor_loss(*CSR, [0], [[1.0]], dropout=0.5)
    u = UnsupervisedGraphsage.__new__(UnsupervisedGraphsage)
    u.aggregator_cls, u.features, u.distributed, u.dropout_rate = MeanAggregator, torch.zeros((5, 3)), False, 0.5
    with pytest.raises(NotImplementedError, match="dropout"):
        u.full_neighbor_minibatch_loss(*CSR, [0], [1])
    with pytest.raises(ValueError, match="dropout"):
        u.full_neighbor_minibatch_loss(*CSR, [0], [1], dropout=2.)


# ---------------------------------------------------------------- the autograd wiring, kernels replaced by the oracle
def _np(t):
    return t.detach().cpu().numpy()


def _fake_sage_gemm(parts, combine=ops.COMBINE_ADD, bias=None, act=ops.ACT_NONE, math=None, out=None, packed=None):
    ys = [a[:, :k] @ w for (a, k, w) in parts]
    y = torch.cat(ys, dim=1) if combine == ops.COMBINE_CONCAT else sum(ys[1:], ys[0])
    if bias is not None:
        y = y + bias
    return torch.relu(y) if act == ops.ACT_RELU else y


def _pm(pos_map):
    a, b, c = pos_map
    return _np(a), (None if b is None else _np(b)), int(c)


def _fake_csr_aggregate(src, indptr, indices, op, rows=None, out=None, dropout=None, t_slot=None):
    import oracle.full_neighbor as fn
    import oracle.full_neighbor_grad as fg
    rows = None if rows is None else _np(rows)
    if dropout is None:
        if op == "sum":
            return torch.from_numpy(fg.csr_sum(_np(src), _np(indptr), _np(indices).astype(np.int64)))
        return torch.from_numpy(fn.csr_aggregate(_np(src), _np(indptr), _np(indices), op, rows))
    ns, ss, pm = dropout
    if op == "sum":
        return torch.from_numpy(fd.csr_sum_dropout(_np(src), _np(indptr), _np(indices).astype(np.int64), _np(t_slot),
                                                   ns[:3], ss[:3], _pm(pm)))
    return torch.from_numpy(fd.csr_aggregate_dropout(_np(src), _np(indptr), _np(indices), op, ns[:3], ss[:3], _pm(pm),
                                                     rows))


def _fake_transpose(indptr, indices, with_self=False, slots=False):
    a, b, c = fd.csr_transpose_slots(_np(indptr), _np(indices), with_self)
    out = (torch.from_numpy(a), torch.from_numpy(b.astype(np.int32)), torch.from_numpy(c.astype(np.int32)))
    return out if slots else out[:2]


def _fake_max_backward(z, m, dm, indptr, indices, t_indptr, t_indices, s=None, out=None):
    import oracle.full_neighbor_grad as fg
    return torch.from_numpy(fg.max_backward(_np(z), _np(m), _np(dm), _np(indptr), _np(indices))[1])


def _fake_embedding_grad(lists, n_rows, d, out=None, sites=None):
    import oracle.full_neighbor_grad as fg
    (ids, g, group, scale), = lists
    return torch.from_numpy(fg.scatter_rows(_np(g)[:, :d], _np(ids), n_rows))


def _fake_dropout_apply(x, site, rows=None, group=1, scale=1.0, out=None, accumulate=False, pos_ids=None):
    n = x.shape[0]
    pos = np.arange(n) if pos_ids is None else _np(pos_ids)
    y = torch.from_numpy(fd._drop(_np(x), tuple(site[:3]), pos))
    if out is not None:
        out.copy_(y)
        return out
    return y


def _fake_l2_(x):
    x.copy_(x / torch.sqrt(torch.clamp((x * x).sum(1, keepdim=True), min=1e-12)))
    return x


@pytest.fixture()
def cpu_kernels(monkeypatch):
    monkeypatch.setattr(ops, "sage_gemm", _fake_sage_gemm)
    monkeypatch.setattr(ops, "csr_aggregate", _fake_csr_aggregate)
    monkeypatch.setattr(ops, "csr_transpose", _fake_transpose)
    monkeypatch.setattr(ops, "csr_max_backward", _fake_max_backward)
    monkeypatch.setattr(ops, "embedding_grad", _fake_embedding_grad)
    monkeypatch.setattr(ops, "dropout_apply", _fake_dropout_apply)
    monkeypatch.setattr(ops, "l2_normalize_rows_", _fake_l2_)
    monkeypatch.setattr(ops, "gather_rows", lambda src, ids, out=None: src[ids.long()].clone())
    monkeypatch.setattr(torch.cuda, "is_current_stream_capturing", lambda: False)


def oracle_dicts(model):
    out = []
    for a in model.aggregators:
        d = dict(type=model.aggregator_type, **{k: _np(v) for k, v in a.vars.items()})
        if hasattr(a, "mlp_layers"):
            d.update(mlp_weights=_np(a.mlp_layers[0].vars["weights"]), mlp_bias=_np(a.mlp_layers[0].vars["bias"]))
        out.append(d)
    return out


def _model(kind, concat, d, N, F, r, rate=0.):
    feats = np.vstack([r.randn(N, F).astype(np.float32), np.zeros((1, F), np.float32)])
    infos = [gs.SAGEInfo("node", None, 3, 8), gs.SAGEInfo("node", None, 3, 8)]
    model = SupervisedGraphsage(3, {"dropout": rate}, torch.from_numpy(feats), torch.zeros((N + 1, 3), dtype=torch.int32),
                                None, infos, concat=concat, aggregator_type=kind, identity_dim=d, weight_decay=0.01,
                                device="cpu", dropout_seed=77)
    model.aggregator_type = kind
    for a in model.aggregators:
        a.math = ops.MATH_FP32_SIMT
    return model


@pytest.mark.parametrize("kind,concat,d", [("mean", True, 0), ("gcn", False, 16), ("maxpool", True, 16),
                                           ("meanpool", False, 0)])
def test_autograd_wiring_matches_the_oracle(cpu_kernels, kind, concat, d):
    r = np.random.RandomState(11)
    indptr, indices = messy_graph(seed=5)
    N, C = len(indptr) - 1, 3
    model = _model(kind, concat, d, N, 6, r, rate=0.5)
    model.dropout_counter = 9
    node_ids = np.array([1, 4, 4, 7, 2, 20], np.int64)
    labels = np.eye(C)[r.randint(0, C, len(node_ids))]
    loss = model.full_neighbor_loss(indptr, indices, node_ids, labels, dropout=model.dropout_rate)
    plan = full_neighbor_site_plan(kind, 2, head=True)
    assert model.dropout_counter == 9 + len(plan)
    loss.backward()
    sites = fd.sites(kind, 2, True, 77, 9, 0.5)
    rl, grads, head, demb = fd.full_neighbor_loss_grads(_np(model.features), indptr, indices, oracle_dicts(model), concat,
                                                        node_ids, labels, _np(model.node_pred_vars["weights"]),
                                                        _np(model.node_pred_vars["bias"]), sites, False, 0.01, d)
    assert abs(float(loss.detach()) - rl) < 1e-5

    def close(t, ref, what):
        assert t.grad is not None, what
        assert np.abs(_np(t.grad) - ref).max() <= 1e-4 * max(1.0, np.abs(ref).max()), what
    for a, g in zip(model.aggregators, grads):
        for k, v in a.vars.items():
            close(v, g[k], k)
        if hasattr(a, "mlp_layers"):
            close(a.mlp_layers[0].vars["weights"], g["mlp_weights"], "mlp_weights")
            close(a.mlp_layers[0].vars["bias"], g["mlp_bias"], "mlp_bias")
    close(model.node_pred_vars["weights"], head["weights"], "head")
    if d:
        close(model.embeds, demb, "embeds")


@pytest.mark.parametrize("kind", ["mean", "gcn", "maxpool", "meanpool"])
def test_rate_zero_is_dropout_none_and_leaves_the_counter(cpu_kernels, kind):
    r = np.random.RandomState(12)
    indptr, indices = messy_graph(seed=6)
    N = len(indptr) - 1
    model = _model(kind, kind != "gcn", 0, N, 6, r)
    ids = np.array([1, 4, 4, 7, 2, 20])
    a = model.full_neighbor_outputs(indptr, indices, ids)
    b = model.full_neighbor_outputs(indptr, indices, ids, dropout=0.)
    assert torch.equal(a, b) and model.dropout_counter == 0
    c = model.full_neighbor_outputs(indptr, indices, ids, dropout=0.5)
    assert not torch.equal(a, c) and model.dropout_counter == len(full_neighbor_site_plan(kind, 2))
    # inference never drops
    assert torch.equal(model.full_neighbor_embeddings(indptr, indices, ids), a.detach())


@pytest.mark.parametrize("kind", ["mean", "gcn", "maxpool", "meanpool"])
def test_minibatch_wiring_equals_the_whole_graph(cpu_kernels, monkeypatch, kind):
    """With the oracle's blocks standing in for ops.csr_blocks, the minibatch rows equal the whole-graph rows."""
    from oracle.full_neighbor_blocks import csr_blocks

    class _B(object):
        pass

    def fake_blocks(indptr, indices, ids, L):
        out = []
        for b in csr_blocks(_np(indptr), _np(indices), _np(ids), L):
            o = _B()
            o.src_ids, o.indptr = torch.from_numpy(b["src_ids"]), torch.from_numpy(b["indptr"])
            o.indices, o.rows = torch.from_numpy(b["indices"]), torch.from_numpy(b["rows"])
            out.append(o)
        return out
    monkeypatch.setattr(ops, "csr_blocks", fake_blocks)
    monkeypatch.setattr(ops, "gather_rows_f32", lambda src, ids, out=None: src[ids.long()].float().clone())
    r = np.random.RandomState(13)
    indptr, indices = messy_graph(seed=8)
    N = len(indptr) - 1
    model = _model(kind, kind != "gcn", 0, N, 6, r)
    ids = np.array([1, 4, 4, 7, 23, 20])
    model.dropout_counter = 5
    whole = model.full_neighbor_outputs(indptr, indices, ids, dropout=0.4)
    model.dropout_counter = 5
    mini = model.full_neighbor_minibatch_outputs(indptr, indices, ids, dropout=0.4)
    assert torch.equal(whole, mini)
