"""Aggregation over weighted edges without a GPU: oracle/weighted.py against a dense float64 restatement and float64
torch autograd, all-one weights against the unweighted oracles bit for bit, blocks and sampled blocks against the
whole graph bit for bit, the autograd wiring of full_neighbor_training with the oracle standing in for the kernels (TEST
mocks only: the product has no such path), and the argument checks and refusals."""
import numpy as np
import pytest
import torch

import graphsage_b200 as gs
from graphsage_b200 import ops
from graphsage_b200.supervised_models import SupervisedGraphsage
from oracle import full_neighbor as fn
from oracle import full_neighbor_grad as fg
from oracle import weighted as ow
from test_full_neighbor_train_cpu import _agg_dicts, _bare_model, messy_graph


def edge_weights(r, n, kind="random"):
    """fp32 weights: random, with zeros and negatives, or all one, or small integers (exact products: max ties)."""
    if kind == "one":
        return np.ones(n, np.float32)
    if kind == "int":
        return r.randint(-1, 3, size=n).astype(np.float32)
    w = (r.randn(n) * 2).astype(np.float32)
    w[::7] = 0
    w[3::11] = -np.abs(w[3::11])
    return w


# ---------------------------------------------------------------- the reductions
@pytest.mark.parametrize("op", ["mean", "mean_self", "max"])
@pytest.mark.parametrize("rows", [None, "subset"])
def test_oracle_matches_the_dense_float64_formula(op, rows):
    r = np.random.RandomState(1)
    indptr, indices = messy_graph(seed=2)
    N = len(indptr) - 1
    x = r.randn(N + 1, 6).astype(np.float32)
    w = edge_weights(r, len(indices))
    rr = None if rows is None else np.array([0, 3, 2, -1, N, N + 7, 5, 5])
    got = ow.csr_aggregate(x, indptr, indices, op, rr, w)
    ref = ow.dense_reference(x, indptr, indices, op, rr, w)
    assert np.abs(got - ref).max() <= 1e-5 * max(1.0, np.abs(ref).max())


@pytest.mark.parametrize("op", ["mean", "mean_self", "max"])
def test_all_one_weights_give_the_unweighted_oracle_bit_for_bit(op):
    r = np.random.RandomState(2)
    indptr, indices = messy_graph(seed=4)
    N = len(indptr) - 1
    x = r.randn(N + 1, 5).astype(np.float32)
    one = np.ones(len(indices), np.float32)
    assert np.array_equal(ow.csr_aggregate(x, indptr, indices, op, None, one), fn.csr_aggregate(x, indptr, indices, op))
    g = r.randn(N + 1, 5).astype(np.float32)
    for with_self in (False, True):
        assert np.array_equal(ow.mean_backward(g, indptr, indices, with_self, one),
                              fg.mean_backward(g, indptr, indices, with_self))
    z = r.randint(0, 3, size=(N + 1, 5)).astype(np.float32)
    m = fn.csr_aggregate(z, indptr, indices, "max")
    for a, b in zip(ow.max_backward(z, m, g, indptr, indices, one), fg.max_backward(z, m, g, indptr, indices)):
        assert np.array_equal(a, b)


def test_a_weighted_message_is_rounded_before_the_sum():
    # fl(w x) then + : 1 + fl(3 * (1/3)) differs from the fused 1 + 3 * (1/3) in the last bit for some values; the rule is
    # the product rounded first, which numpy's float32 multiply does
    x = np.array([[1.0], [np.float32(1) / np.float32(3)], [0.0]], np.float32)
    indptr, indices = np.array([0, 2, 2], np.int64), np.array([0, 1], np.int32)
    w = np.array([1.0, 3.0], np.float32)
    got = ow.csr_aggregate(x, indptr, indices, "mean", [0], w)
    assert got[0, 0] == (np.float32(1) + np.float32(w[1] * x[1, 0])) / np.float32(2)


def test_transpose_weights_follow_their_forward_entries():
    r = np.random.RandomState(3)
    indptr, indices = messy_graph(seed=5)
    w = edge_weights(r, len(indices))
    for with_self in (False, True):
        t_indptr, t_indices = fg.csr_transpose(indptr, indices, with_self)
        tw = ow.transpose_weights(indptr, indices, w, with_self)
        eptr, eidx = fg.effective_csr(indptr, indices, with_self)
        ew = ow.effective_weights(indptr, w, with_self)
        # each (destination, source row) pair carries the multiset of weights of the effective entries it came from
        for j in range(len(t_indptr) - 1):
            got = sorted(zip(t_indices[t_indptr[j]:t_indptr[j + 1]].tolist(), tw[t_indptr[j]:t_indptr[j + 1]].tolist()))
            want = sorted((i, float(ew[k])) for i in range(len(eptr) - 1) for k in range(eptr[i], eptr[i + 1])
                          if eidx[k] == j)
            assert got == want


# ---------------------------------------------------------------- blocks
CONCAT = {"mean": True, "gcn": False, "maxpool": True, "meanpool": False}


@pytest.mark.parametrize("kind", ["mean", "gcn", "maxpool", "meanpool"])
@pytest.mark.parametrize("L", [1, 2])
def test_blocks_and_sampled_blocks_give_the_whole_graph_rows(kind, L):
    r = np.random.RandomState(4)
    indptr, indices = messy_graph(seed=6)
    N = len(indptr) - 1
    feats = np.vstack([r.randn(N, 5).astype(np.float32), np.zeros((1, 5), np.float32)])
    aggs = _agg_dicts(kind, [5] + [4] * L, CONCAT[kind], r)
    w = edge_weights(r, len(indices))
    seeds = np.array([0, 3, 5, 5, 2, -4, N + 1, 11])
    whole = ow.embeddings(feats, indptr, indices, w, aggs, CONCAT[kind], seeds)
    blocks = ow.embeddings(feats, indptr, indices, w, aggs, CONCAT[kind], seeds, mode="blocks")
    big = int(np.diff(indptr).max())                          # fanouts >= every degree: every entry is kept
    sampled = ow.embeddings(feats, indptr, indices, w, aggs, CONCAT[kind], seeds, mode="sampled", fanouts=[big] * L,
                            seed=5, call=2)
    assert np.array_equal(whole, blocks) and np.array_equal(whole, sampled)
    # the weights matter: unweighted rows differ
    assert not np.array_equal(whole, fn.full_neighbor_embeddings(feats, indptr, indices, aggs, CONCAT[kind], seeds))


def test_sampled_block_weights_follow_the_raw_entries():
    from oracle.sampled_blocks_dropout import entry_offsets
    indptr, indices = messy_graph(seed=7)
    w = np.arange(len(indices), dtype=np.float32)             # weight = the entry's raw CSR position
    blocks, offs = entry_offsets(indptr, indices, np.array([2, 4, 9]), [3, 2], 7, 1)
    for b, o in zip(blocks, offs):
        bw = ow.block_weights(indptr, w, b, o)
        cnt = np.diff(b["indptr"])
        g = np.repeat(b["src_ids"][:len(cnt)].astype(np.int64), cnt)
        assert np.array_equal(bw, (indptr[g] + o).astype(np.float32))


# ---------------------------------------------------------------- gradients against float64 autograd
def _torch_weighted(feats, indptr, indices, w, aggs, concat, node_ids, pred_w, pred_b, labels, wd, d):
    """loss of the weighted layer loop in float64 torch from dense weighted adjacencies (amax splits ties evenly)."""
    N = len(indptr) - 1
    W = np.zeros((N + 1, N + 1))                              # weighted effective adjacency
    cnt = np.zeros(N + 1)
    lists = []
    for i in range(N + 1):
        if i < N and indptr[i + 1] > indptr[i]:
            ids = indices[indptr[i]:indptr[i + 1]].astype(np.int64)
            ids = np.where((ids < 0) | (ids > N), N, ids)
            ws = w[indptr[i]:indptr[i + 1]].astype(np.float64)
        else:
            ids, ws = np.array([N]), np.ones(1)
        np.add.at(W[i], ids, ws)
        cnt[i] = len(ids)
        lists.append((ids, ws))
    width = max(len(a) for a, _ in lists)
    idx = torch.tensor(np.array([np.pad(a, (0, width - len(a))) for a, _ in lists]))
    wts = torch.tensor(np.array([np.pad(b, (0, width - len(b))) for _, b in lists]))
    mask = torch.tensor(np.array([np.arange(width) < len(a) for a, _ in lists]))
    A = torch.from_numpy(W / cnt[:, None])
    As = torch.from_numpy((W + np.eye(N + 1)) / (cnt + 1)[:, None])
    emb = torch.from_numpy(feats[:, :d].astype(np.float64)).requires_grad_(True) if d else None
    h = torch.from_numpy(feats.astype(np.float64))
    if d:
        h = torch.cat([emb, h[:, d:]], dim=1)
    params = [{k: torch.from_numpy(v.astype(np.float64)).requires_grad_(True) for k, v in a.items() if k != "type"}
              for a in aggs]
    L = len(aggs)
    for l, (a, p) in enumerate(zip(aggs, params)):
        if a["type"] == "gcn":
            y = As @ h @ p["weights"]
        else:
            if a["type"] == "mean":
                nb = A @ h
            else:
                z = torch.relu(h @ p["mlp_weights"] + p["mlp_bias"])
                if a["type"] == "maxpool":
                    nb = torch.where(mask.unsqueeze(2), wts.unsqueeze(2) * z[idx],
                                     torch.tensor(-np.inf, dtype=z.dtype)).amax(dim=1)
                else:
                    nb = A @ z
            fs, fnb = h @ p["self_weights"], nb @ p["neigh_weights"]
            y = torch.cat([fs, fnb], 1) if concat else fs + fnb
        h = y[torch.from_numpy(np.asarray(node_ids, np.int64))] if l == L - 1 else torch.relu(y)
    out = h / torch.sqrt(torch.clamp((h * h).sum(1, keepdim=True), min=1e-12))
    Wp = torch.from_numpy(pred_w.astype(np.float64)).requires_grad_(True)
    b = torch.from_numpy(pred_b.astype(np.float64)).requires_grad_(True)
    loss = (-(torch.from_numpy(labels) * torch.log_softmax(out @ Wp + b, 1)).sum(1)).mean()
    decayed = [Wp, b] + [v for p in params for k, v in p.items() if not k.startswith("mlp")]
    loss = loss + wd * 0.5 * sum((v * v).sum() for v in decayed)
    loss.backward()
    return float(loss.detach()), [{k: v.grad.numpy() for k, v in p.items()} for p in params], \
        {"weights": Wp.grad.numpy(), "bias": b.grad.numpy()}, (emb.grad.numpy() if d else None)


GRAD_CASES = [  # kind, concat, identity_dim, layers, weights ("int": exact products, max ties), integer features
    ("mean", True, 0, 2, "random", False), ("mean", False, 16, 2, "random", False), ("gcn", False, 16, 2, "random", False),
    ("maxpool", True, 0, 2, "random", False), ("maxpool", True, 16, 2, "int", True), ("maxpool", False, 0, 3, "int", True),
    ("meanpool", True, 16, 2, "random", False), ("mean", True, 0, 3, "int", False),
]


@pytest.mark.parametrize("kind,concat,d,L,wkind,integer", GRAD_CASES)
def test_oracle_gradients_equal_float64_autograd(kind, concat, d, L, wkind, integer):
    r = np.random.RandomState(7)
    indptr, indices = messy_graph(seed=3)
    N, F, C = len(indptr) - 1, 5, 3
    x = r.randint(0, 3, size=(N + 1, F)).astype(np.float32) if integer else r.randn(N + 1, F).astype(np.float32)
    x[N] = 0
    feats = np.concatenate([r.randn(N + 1, d).astype(np.float32), x], 1) if d else x
    dims = [d + F] + [4] * L
    aggs = _agg_dicts(kind, dims, concat, r, integer)
    w = edge_weights(r, len(indices), wkind)
    node_ids = np.array([0, 3, 5, 5, 9, 2, 11, 3, 23], np.int64)
    out_w = dims[-1] * (2 if concat and kind != "gcn" else 1)
    pred_w, pred_b = (r.randn(out_w, C) * 0.5).astype(np.float32), (r.randn(C) * 0.1).astype(np.float32)
    labels = np.eye(C)[r.randint(0, C, len(node_ids))]
    loss, grads, head, demb = ow.loss_grads(feats, indptr, indices, w, aggs, concat, node_ids, labels, pred_w, pred_b,
                                            False, 0.01, d)
    rl, rgrads, rhead, rdemb = _torch_weighted(feats, indptr, indices, w, aggs, concat, node_ids, pred_w, pred_b, labels,
                                               0.01, d)
    assert abs(loss - rl) < 1e-5 * max(1, abs(rl))

    def close(a, b, what):
        assert a.shape == b.shape, what
        assert np.abs(a - b).max() <= 1e-4 * max(1.0, np.abs(b).max()), (what, np.abs(a - b).max())
    for l, (g, rg) in enumerate(zip(grads, rgrads)):
        assert set(g) == set(rg)
        for k in g:
            close(g[k], rg[k], (l, k))
    close(head["weights"], rhead["weights"], "head")
    if d:
        close(demb, rdemb, "embeddings")
    if wkind == "int" and kind == "maxpool":               # exact weighted ties occurred and were split
        z = np.maximum(feats @ aggs[0]["mlp_weights"] + aggs[0]["mlp_bias"], 0).astype(np.float32)
        m = ow.csr_aggregate(z, indptr, indices, "max", None, w)
        eptr, eidx = fg.effective_csr(indptr, indices)
        ew = ow.effective_weights(indptr, w)
        ties = [((ew[eptr[i]:eptr[i + 1], None] * z[eidx[eptr[i]:eptr[i + 1]]]) == m[i]).sum(0).max()
                for i in range(N + 1)]
        assert max(ties) >= 2


def test_max_backward_routes_w_dm_over_ties():
    # row 0 = {1, 2, 3} with weights (2, 1, -1) and z = (1, 2, 0): weighted terms (2, 2, -0), the max 2 tied twice
    indptr, indices = np.array([0, 3, 3, 3, 3], np.int64), np.array([1, 2, 3], np.int32)
    w = np.array([2.0, 1.0, -1.0], np.float32)
    z = np.array([[0.0], [1.0], [2.0], [0.0], [0.0]], np.float32)
    m = ow.csr_aggregate(z, indptr, indices, "max", None, w)
    assert m[0, 0] == 2.0
    dm = np.zeros_like(z)
    dm[0] = 3.0
    s, dz = ow.max_backward(z, m, dm, indptr, indices, w)
    assert s[0, 0] == 1.5                                   # ties: z1 (2 * 1) and z2 (1 * 2); z3 = 0 gives 0
    assert dz[1, 0] == 3.0 and dz[2, 0] == 1.5 and dz[3, 0] == 0.0   # w * dm / ties; z3 is not a max (and <= 0)


# ---------------------------------------------------------------- the autograd wiring, kernels replaced by the oracle
def _np(t):
    return t.detach().cpu().numpy()


def _slots(indptr, indices, with_self):
    """t_slot of csr_transpose(..., slots=True) from the oracle's effective CSR."""
    N = len(indptr) - 1
    slot = []
    for i in range(N + 1):
        c = int(indptr[i + 1] - indptr[i]) if i < N else 0
        slot += list(range(c)) if c > 0 else [-1]
        slot += [-2] if with_self else []
    _, eidx = fg.effective_csr(indptr, indices, with_self)
    return np.array(slot, np.int32)[np.argsort(eidx, kind="stable")]


@pytest.fixture()
def oracle_kernels(monkeypatch):
    from test_full_neighbor_train_cpu import _fake_embedding_grad, _fake_l2_, _fake_sage_gemm

    def aggregate(src, indptr, indices, op, rows=None, out=None, weights=None):
        w = None if weights is None else _np(weights)
        if op == "sum":
            return torch.from_numpy(ow.csr_sum(_np(src), _np(indptr), _np(indices).astype(np.int64), w))
        return torch.from_numpy(ow.csr_aggregate(_np(src), _np(indptr), _np(indices), op,
                                                 None if rows is None else _np(rows), w))

    def transpose(indptr, indices, with_self=False, slots=False):
        t_indptr, t_indices = fg.csr_transpose(_np(indptr), _np(indices), with_self)
        out = (torch.from_numpy(t_indptr), torch.from_numpy(t_indices.astype(np.int32)))
        return out + (torch.from_numpy(_slots(_np(indptr), _np(indices), with_self)),) if slots else out

    def max_backward(z, m, dm, indptr, indices, t_indptr, t_indices, s=None, out=None, weights=None, t_weights=None):
        return torch.from_numpy(ow.max_backward(_np(z), _np(m), _np(dm), _np(indptr), _np(indices), _np(weights))[1])

    monkeypatch.setattr(ops, "sage_gemm", _fake_sage_gemm)
    monkeypatch.setattr(ops, "csr_aggregate", aggregate)
    monkeypatch.setattr(ops, "csr_transpose", transpose)
    monkeypatch.setattr(ops, "csr_max_backward", max_backward)
    monkeypatch.setattr(ops, "embedding_grad", _fake_embedding_grad)
    monkeypatch.setattr(ops, "l2_normalize_rows_", _fake_l2_)
    monkeypatch.setattr(ops, "gather_rows", lambda src, ids, out=None: src[ids.long()].clone())
    monkeypatch.setattr(ops, "require_cuda", lambda *t: None)     # csr_transpose_weights' torch gathers run on the CPU
    monkeypatch.setattr(torch.cuda, "is_current_stream_capturing", lambda: False)


def _oracle_dicts(model):
    out = []
    for a in model.aggregators:
        d = dict(type=model.aggregator_type, **{k: _np(v) for k, v in a.vars.items()})
        if hasattr(a, "mlp_layers"):
            d.update(mlp_weights=_np(a.mlp_layers[0].vars["weights"]), mlp_bias=_np(a.mlp_layers[0].vars["bias"]))
        out.append(d)
    return out


@pytest.mark.parametrize("kind,concat,d", [("mean", True, 0), ("gcn", False, 16), ("maxpool", True, 16),
                                           ("meanpool", False, 0)])
def test_autograd_wiring_matches_the_oracle(oracle_kernels, kind, concat, d):
    r = np.random.RandomState(11)
    indptr, indices = messy_graph(seed=5)
    N, F, C = len(indptr) - 1, 6, 3
    feats = np.vstack([r.randn(N, F).astype(np.float32), np.zeros((1, F), np.float32)])
    infos = [gs.SAGEInfo("node", None, 3, 8), gs.SAGEInfo("node", None, 3, 8)]
    model = SupervisedGraphsage(C, {}, torch.from_numpy(feats), torch.zeros((N + 1, 3), dtype=torch.int32), None, infos,
                                concat=concat, aggregator_type=kind, identity_dim=d, weight_decay=0.01, device="cpu")
    model.aggregator_type = kind
    for a in model.aggregators:
        a.math = ops.MATH_FP32_SIMT
    w = edge_weights(r, len(indices))
    node_ids = np.array([1, 4, 4, 7, 2, 20], np.int64)
    labels = np.eye(C)[r.randint(0, C, len(node_ids))]
    loss = model.full_neighbor_loss(indptr, indices, node_ids, labels, edge_weight=w)
    loss.backward()
    rl, grads, head, demb = ow.loss_grads(_np(model.features), indptr, indices, w, _oracle_dicts(model), concat,
                                          node_ids, labels, _np(model.node_pred_vars["weights"]),
                                          _np(model.node_pred_vars["bias"]), False, 0.01, d)
    assert abs(float(loss.detach()) - rl) < 1e-5

    def close(t, ref, what):
        assert t.grad is not None, what
        assert np.abs(_np(t.grad) - ref).max() <= 1e-4 * max(1.0, np.abs(ref).max()), what
    for a, g in zip(model.aggregators, grads):
        for k, v in a.vars.items():
            close(v, g[k], k)
        if hasattr(a, "mlp_layers"):
            close(a.mlp_layers[0].vars["weights"], g["mlp_weights"], "mlp_weights")
    close(model.node_pred_vars["weights"], head["weights"], "head")
    if d:
        close(model.embeds, demb, "embeds")
    # the transposes and their weights are cached, keyed by the weight tensor too
    g0 = model._full_neighbor_graph
    assert g0.weights is not None and g0._tw
    wt = g0.weights
    from graphsage_b200 import full_neighbor_training as fnt
    assert fnt.full_neighbor_graph(model, g0.indptr, g0.indices, wt) is g0
    wt.mul_(1)                                                              # a new _version: rebuilt
    assert fnt.full_neighbor_graph(model, g0.indptr, g0.indices, wt) is not g0
    # embeddings (no autograd) are the training forward
    emb = model.full_neighbor_embeddings(indptr, indices, node_ids, edge_weight=w)
    out = model.full_neighbor_outputs(indptr, indices, node_ids, edge_weight=w)
    assert torch.equal(emb, out.detach())


# ---------------------------------------------------------------- argument checks and refusals
def test_edge_weight_checks_and_refusals():
    m = _bare_model()
    indptr, indices = np.array([0, 1, 2, 2, 3], np.int64), np.array([1, 0, 2], np.int32)
    with pytest.raises(ValueError, match="one weight per CSR entry"):
        m.full_neighbor_outputs(indptr, indices, [0], edge_weight=np.ones(2, np.float32))
    with pytest.raises(ValueError, match="one weight per CSR entry"):
        m.full_neighbor_outputs(indptr, indices, [0], edge_weight=torch.ones((3, 1)))
    with pytest.raises(TypeError, match="float32"):
        m.full_neighbor_outputs(indptr, indices, [0], edge_weight=np.ones(3))
    with pytest.raises(TypeError, match="float32"):
        m.full_neighbor_outputs(indptr, indices, [0], edge_weight=torch.ones(3, dtype=torch.float64))
    for call in (lambda: m.full_neighbor_outputs(indptr, indices, [0], dropout=0.5, edge_weight=np.ones(3, np.float32)),
                 lambda: m.full_neighbor_train_step(indptr, indices, [0], [[1.0]], dropout=0.3,
                                                    edge_weight=np.ones(3, np.float32))):
        with pytest.raises(NotImplementedError, match="edge_weight with training dropout"):
            call()
    # the whole-graph refusals of host and int8 tables keep their own messages
    from graphsage_b200.host_features import HostFeatures
    h = _bare_model()
    h.features = HostFeatures.__new__(HostFeatures)
    with pytest.raises(NotImplementedError, match="it reads the whole table"):
        h.full_neighbor_outputs(indptr, indices, [0], edge_weight=np.ones(3, np.float32))


def test_max_backward_takes_both_weight_arrays_or_neither():
    z = torch.zeros((3, 2))
    with pytest.raises(ValueError, match="both weights and t_weights"):
        ops.csr_max_backward(z, z, z, torch.zeros(3, dtype=torch.int64), torch.zeros(0, dtype=torch.int32),
                             torch.zeros(4, dtype=torch.int64), torch.zeros(3, dtype=torch.int32),
                             weights=torch.ones(0))
