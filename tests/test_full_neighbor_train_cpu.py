"""Full-batch training over whole neighbourhoods without a GPU: the backward contract (oracle/full_neighbor_grad.py)
against float64 torch autograd of oracle/full_neighbor.py's formula, the transpose against a dense adjacency, the
refusals, and the autograd wiring of full_neighbor_training with torch stand-ins for the kernels (TEST mocks only: the
product has no such path)."""
import numpy as np
import pytest
import torch

import graphsage_b200 as gs
from graphsage_b200 import full_neighbor_training as fnt
from graphsage_b200 import ops
from graphsage_b200.aggregators import MeanAggregator, SeqAggregator
from graphsage_b200.supervised_models import SupervisedGraphsage
from oracle import full_neighbor as fn
from oracle import full_neighbor_grad as fg


# ---------------------------------------------------------------- graphs
def messy_graph(N=24, seed=0):
    """A CSR with empty rows, duplicate entries, self loops and out-of-range entries (clamped to the dummy N); node N - 1 is
    nobody's neighbour."""
    r = np.random.RandomState(seed)
    rows = []
    for i in range(N):
        deg = 0 if i % 7 == 3 else r.randint(1, 6)
        e = list(r.randint(0, N - 1, size=deg))
        if i % 5 == 0 and deg:
            e += [i, e[0]]                                # a self loop and a duplicate
        if i % 6 == 1:
            e += [N + 3, -2]                              # out of range: reads the dummy row
        rows.append(e)
    rows[2] = list(range(N - 1)) * 2                      # one long row
    indptr = np.zeros(N + 1, np.int64)
    indptr[1:] = np.cumsum([len(e) for e in rows])
    return indptr, np.array([x for e in rows for x in e], dtype=np.int32)


def dense_adjacency(indptr, indices, with_self=False):
    """float64 [N+1, N+1] entry counts of the effective rows, built from the raw CSR."""
    N = len(indptr) - 1
    A = np.zeros((N + 1, N + 1))
    for i in range(N):
        if indptr[i + 1] > indptr[i]:
            for d in indices[indptr[i]:indptr[i + 1]]:
                A[i, d if 0 <= d <= N else N] += 1
        else:
            A[i, N] += 1
    A[N, N] += 1
    return A + np.eye(N + 1) if with_self else A


@pytest.mark.parametrize("with_self", [False, True])
def test_transpose_equals_the_dense_adjacency(with_self):
    indptr, indices = messy_graph()
    t_indptr, t_indices = fg.csr_transpose(indptr, indices, with_self)
    A = dense_adjacency(indptr, indices, with_self)
    N = len(indptr) - 1
    assert t_indptr[0] == 0 and t_indptr[-1] == A.sum()
    for j in range(N + 1):
        col = t_indices[t_indptr[j]:t_indptr[j + 1]]
        assert np.all(np.diff(col) >= 0)                                       # ascending source rows
        assert np.array_equal(np.bincount(col, minlength=N + 1), A[:, j])     # with multiplicities


def test_transpose_of_an_edgeless_graph_is_the_dummy_column():
    t_indptr, t_indices = fg.csr_transpose(np.zeros(4, np.int64), np.zeros(0, np.int32))
    assert list(t_indptr) == [0, 0, 0, 0, 4] and list(t_indices) == [0, 1, 2, 3]


@pytest.mark.parametrize("with_self", [False, True])
def test_mean_backward_is_the_transposed_normalised_adjacency(with_self):
    indptr, indices = messy_graph(seed=1)
    A = dense_adjacency(indptr, indices, with_self)
    g = np.random.RandomState(2).randn(A.shape[0], 5).astype(np.float32)
    got = fg.mean_backward(g, indptr, indices, with_self)
    ref = (A / A.sum(axis=1, keepdims=True)).T @ g
    assert np.abs(got - ref).max() < 1e-5
    if not with_self:                                                          # (with it, every node reads itself)
        unread = np.nonzero(A.sum(axis=0) == 0)[0]
        assert len(unread) and np.all(got[unread] == 0)                        # nobody's neighbour: exactly 0


def test_max_backward_splits_ties_evenly_and_applies_the_relu():
    indptr = np.array([0, 3, 5, 5], np.int64)                                  # row 2 empty: {N}
    indices = np.array([1, 1, 0, 0, 2], np.int32)                              # row 0 reads node 1 twice
    z = np.array([[2., 0.], [2., 1.], [0., 1.], [3., 0.]], np.float32)
    m = fn.csr_aggregate(z, indptr, indices, "max")
    dm = np.ones_like(m)
    s, dz = fg.max_backward(z, m, dm, indptr, indices)
    third = np.float32(1) / np.float32(3)
    assert np.array_equal(s[0], np.float32([third, 0.5]))   # column 0: entries 1, 1, 0 all equal 2; column 1: 1, 1 tie
    # node 0: rows 0 (1/3) and 1 (alone at the max); node 1: twice in row 0; node 2: z = 0; the dummy: rows 2 and 3
    assert np.array_equal(dz[:, 0], np.float32([third + np.float32(1), third + third, 0, 2]))
    assert dz[0, 1] == 0 and dz[3, 1] == 0 and dz[2, 1] == 1    # z == 0: the ReLU stops the gradient


# ---------------------------------------------------------------- float64 autograd of the formula
def _agg_dicts(kind, dims, concat, r, integer=False):
    aggs = []
    for l in range(len(dims) - 1):
        din = dims[l] * (2 if concat and l and kind != "gcn" else 1)
        w = (lambda *s: r.randint(-1, 2, size=s).astype(np.float32)) if integer else \
            (lambda *s: (r.randn(*s) * 0.5).astype(np.float32))
        if kind == "gcn":
            aggs.append(dict(type="gcn", weights=w(din, dims[l + 1])))
        elif kind == "mean":
            aggs.append(dict(type="mean", self_weights=w(din, dims[l + 1]), neigh_weights=w(din, dims[l + 1])))
        else:
            hid = 8
            aggs.append(dict(type=kind, mlp_weights=w(din, hid), mlp_bias=(w(hid) if integer else w(hid) * 0.1),
                             self_weights=w(din, dims[l + 1]), neigh_weights=w(hid, dims[l + 1])))
    return aggs


def _torch_formula(feats, indptr, indices, aggs, concat, node_ids, pred_w, pred_b, labels, sigmoid, wd, d):
    """loss of the layer loop in float64 torch from dense adjacencies (amax splits ties evenly, like TF)."""
    N = len(indptr) - 1
    A = torch.from_numpy(dense_adjacency(indptr, indices))
    As = torch.from_numpy(dense_adjacency(indptr, indices, True))
    lists = [np.nonzero(A[i].numpy())[0] for i in range(N + 1)]
    reps = [np.repeat(lst, A[i].numpy()[lst].astype(int)) for i, lst in enumerate(lists)]
    width = max(len(x) for x in reps)
    idx = torch.tensor(np.array([np.pad(x, (0, width - len(x))) for x in reps]))
    mask = torch.tensor(np.array([np.arange(width) < len(x) for x in reps]))
    emb = torch.from_numpy(feats[:, :d].astype(np.float64)).requires_grad_(True) if d else None
    h = torch.from_numpy(feats.astype(np.float64))
    if d:
        h = torch.cat([emb, h[:, d:]], dim=1)
    params = [{k: torch.from_numpy(v.astype(np.float64)).requires_grad_(True) for k, v in a.items() if k != "type"}
              for a in aggs]
    ids = torch.from_numpy(np.asarray(node_ids, np.int64))
    L = len(aggs)
    for l, (a, p) in enumerate(zip(aggs, params)):
        last = l == L - 1
        if a["type"] == "gcn":
            y = (As / As.sum(1, keepdim=True)) @ h @ p["weights"]
        else:
            if a["type"] == "mean":
                nb = (A / A.sum(1, keepdim=True)) @ h
            else:
                z = torch.relu(h @ p["mlp_weights"] + p["mlp_bias"])
                if a["type"] == "maxpool":
                    nb = torch.where(mask.unsqueeze(2), z[idx], torch.tensor(-np.inf, dtype=z.dtype)).amax(dim=1)
                else:
                    nb = (A / A.sum(1, keepdim=True)) @ z
            fs, fnb = h @ p["self_weights"], nb @ p["neigh_weights"]
            y = torch.cat([fs, fnb], 1) if concat else fs + fnb
        h = y[ids] if last else torch.relu(y)
    out = h / torch.sqrt(torch.clamp((h * h).sum(1, keepdim=True), min=1e-12))
    W = torch.from_numpy(pred_w.astype(np.float64)).requires_grad_(True)
    b = torch.from_numpy(pred_b.astype(np.float64)).requires_grad_(True)
    logits = out @ W + b
    lab = torch.from_numpy(labels)
    if sigmoid:
        loss = torch.nn.functional.binary_cross_entropy_with_logits(logits, lab)
    else:
        loss = (-(lab * torch.log_softmax(logits, 1)).sum(1)).mean()
    decayed = [W, b] + [v for p in params for k, v in p.items() if not k.startswith("mlp")]
    loss = loss + wd * 0.5 * sum((v * v).sum() for v in decayed)
    loss.backward()
    return float(loss.detach()), [{k: v.grad.numpy() for k, v in p.items()} for p in params], \
        {"weights": W.grad.numpy(), "bias": b.grad.numpy()}, (emb.grad.numpy() if d else None)


CASES = [  # kind, concat, identity_dim, layers, integer (exact max ties), sigmoid
    ("mean", True, 0, 2, False, False), ("mean", False, 16, 2, False, True),
    ("gcn", False, 0, 2, False, False), ("gcn", True, 16, 2, False, True),
    ("maxpool", True, 0, 2, False, False), ("maxpool", False, 16, 2, False, True),
    ("maxpool", True, 0, 2, True, False), ("meanpool", True, 16, 2, False, False),
    ("meanpool", False, 0, 2, False, True), ("mean", True, 0, 3, False, False), ("maxpool", True, 16, 3, True, True),
]


@pytest.mark.parametrize("kind,concat,d,L,integer,sigmoid", CASES)
def test_oracle_backward_equals_float64_autograd(kind, concat, d, L, integer, sigmoid):
    r = np.random.RandomState(7)
    indptr, indices = messy_graph(seed=3)
    N, F, C = len(indptr) - 1, 5, 3
    x = r.randint(0, 3, size=(N + 1, F)).astype(np.float32) if integer else r.randn(N + 1, F).astype(np.float32)
    x[N] = 0
    feats = np.concatenate([r.randn(N + 1, d).astype(np.float32), x], 1) if d else x
    dims = [d + F] + [4] * L
    aggs = _agg_dicts(kind, dims, concat, r, integer)
    node_ids = np.array([0, 3, 5, 5, 9, 2, 11, 3, 23], np.int64)                # duplicates, an empty row, the long row
    out_w = dims[-1] * (2 if concat and kind != "gcn" else 1)
    pred_w, pred_b = (r.randn(out_w, C) * 0.5).astype(np.float32), (r.randn(C) * 0.1).astype(np.float32)
    labels = (r.rand(len(node_ids), C) > 0.5).astype(np.float64) if sigmoid else np.eye(C)[r.randint(0, C, len(node_ids))]
    wd = 0.01
    loss, grads, head, demb = fg.full_neighbor_loss_grads(feats, indptr, indices, aggs, concat, node_ids, labels, pred_w,
                                                          pred_b, sigmoid, wd, d)
    rl, rgrads, rhead, rdemb = _torch_formula(feats, indptr, indices, aggs, concat, node_ids, pred_w, pred_b, labels,
                                              sigmoid, wd, d)
    assert abs(loss - rl) < 1e-5 * max(1, abs(rl))

    def close(a, b, what):
        assert a.shape == b.shape, what
        assert np.abs(a - b).max() <= 1e-4 * max(1.0, np.abs(b).max()), (what, np.abs(a - b).max())
    for l, (g, rg) in enumerate(zip(grads, rgrads)):
        assert set(g) == set(rg)
        for k in g:
            close(g[k], rg[k], (l, k))
    close(head["weights"], rhead["weights"], "head")
    close(head["bias"], rhead["bias"], "head bias")
    if d:
        close(demb, rdemb, "embeddings")
    # the forward is oracle/full_neighbor.py's, unchanged
    ref = fn.full_neighbor_embeddings(feats, indptr, indices, aggs, concat, node_ids)
    assert ref.shape == (len(node_ids), out_w)


# ---------------------------------------------------------------- refusals (no GPU needed: they fire first)
def _bare_model(kind="mean", **attrs):
    m = SupervisedGraphsage.__new__(SupervisedGraphsage)
    m.aggregator_cls = {"mean": MeanAggregator, "seq": SeqAggregator}[kind]
    m.features = torch.zeros((5, 3))
    m.device = torch.device("cpu")
    m.aggregators = None
    m.distributed, m.dropout_rate = False, 0.
    for k, v in attrs.items():
        setattr(m, k, v)
    return m


CSR = (np.zeros(5, np.int64), np.zeros(0, np.int32))


def test_refusals():
    with pytest.raises(NotImplementedError, match="seq"):
        _bare_model("seq").full_neighbor_train_step(*CSR, [0], [[1.0]])
    m = _bare_model()
    m.features = type("Sharded", (), {"c_table": lambda self: None, "shape": (5, 3)})()
    with pytest.raises(NotImplementedError, match="ShardedFeatures"):
        m.full_neighbor_loss(*CSR, [0], [[1.0]])
    with pytest.raises(NotImplementedError, match="distributed"):
        _bare_model(distributed=True).full_neighbor_outputs(*CSR, [0])
    with pytest.raises(NotImplementedError, match="dropout"):
        _bare_model(dropout_rate=0.5).full_neighbor_train_step(*CSR, [0], [[1.0]])


def test_refuses_csr_of_the_wrong_dtype_or_length():
    m = _bare_model()
    with pytest.raises(TypeError, match="indptr"):
        m.full_neighbor_outputs(np.zeros(5, np.int32), np.zeros(0, np.int32), [0])
    with pytest.raises(TypeError, match="indices"):
        m.full_neighbor_outputs(np.zeros(5, np.int64), np.zeros(0, np.int64), [0])
    with pytest.raises(ValueError, match="N \\+ 1"):
        m.full_neighbor_train_step(np.zeros(4, np.int64), np.zeros(0, np.int32), [0], [[1.0]])


def test_new_ops_have_no_cpu_fallback():
    with pytest.raises(RuntimeError, match="CUDA-only"):
        ops.csr_transpose(torch.zeros(3, dtype=torch.int64), torch.zeros(0, dtype=torch.int32))
    z = torch.zeros((3, 2))
    with pytest.raises(RuntimeError, match="CUDA-only"):
        ops.csr_max_backward(z, z, z, torch.zeros(3, dtype=torch.int64), torch.zeros(0, dtype=torch.int32),
                             torch.zeros(4, dtype=torch.int64), torch.zeros(3, dtype=torch.int32))


# ---------------------------------------------------------------- the autograd wiring, kernels replaced by the oracle
def _np(t):
    return t.detach().cpu().numpy()


def _fake_sage_gemm(parts, combine=ops.COMBINE_ADD, bias=None, act=ops.ACT_NONE, math=None, out=None, packed=None):
    ys = [a[:, :k] @ w for (a, k, w) in parts]
    y = torch.cat(ys, dim=1) if combine == ops.COMBINE_CONCAT else sum(ys[1:], ys[0])
    if bias is not None:
        y = y + bias
    return torch.relu(y) if act == ops.ACT_RELU else y


def _fake_csr_aggregate(src, indptr, indices, op, rows=None, out=None):
    if op == "sum":
        return torch.from_numpy(fg.csr_sum(_np(src), _np(indptr), _np(indices).astype(np.int64)))
    return torch.from_numpy(fn.csr_aggregate(_np(src), _np(indptr), _np(indices), op,
                                             None if rows is None else _np(rows)))


def _fake_transpose(indptr, indices, with_self=False):
    t_indptr, t_indices = fg.csr_transpose(_np(indptr), _np(indices), with_self)
    return torch.from_numpy(t_indptr), torch.from_numpy(t_indices.astype(np.int32))


def _fake_max_backward(z, m, dm, indptr, indices, t_indptr, t_indices, s=None, out=None):
    return torch.from_numpy(fg.max_backward(_np(z), _np(m), _np(dm), _np(indptr), _np(indices))[1])


def _fake_embedding_grad(lists, n_rows, d, out=None, sites=None):
    (ids, g, group, scale), = lists
    return torch.from_numpy(fg.scatter_rows(_np(g)[:, :d], _np(ids), n_rows))


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


@pytest.mark.parametrize("kind,concat,d", [("mean", True, 0), ("gcn", False, 16), ("maxpool", True, 16),
                                           ("meanpool", False, 0)])
def test_autograd_wiring_matches_the_oracle(cpu_kernels, kind, concat, d):
    r = np.random.RandomState(11)
    indptr, indices = messy_graph(seed=5)
    N, F, C = len(indptr) - 1, 6, 3
    feats = np.vstack([r.randn(N, F).astype(np.float32), np.zeros((1, F), np.float32)])
    infos = [gs.SAGEInfo("node", None, 3, 8), gs.SAGEInfo("node", None, 3, 8)]
    adj = torch.zeros((N + 1, 3), dtype=torch.int32)
    model = SupervisedGraphsage(C, {}, torch.from_numpy(feats), adj, None, infos, concat=concat, aggregator_type=kind,
                                identity_dim=d, weight_decay=0.01, device="cpu")
    model.aggregator_type = kind
    for a in model.aggregators:
        a.math = ops.MATH_FP32_SIMT
    node_ids = np.array([1, 4, 4, 7, 2, 20], np.int64)
    labels = np.eye(C)[r.randint(0, C, len(node_ids))]
    loss = model.full_neighbor_loss(indptr, indices, node_ids, labels)
    loss.backward()
    table = _np(model.features)
    rl, grads, head, demb = fg.full_neighbor_loss_grads(table, indptr, indices, oracle_dicts(model), concat, node_ids,
                                                        labels, _np(model.node_pred_vars["weights"]),
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
            close(a.mlp_layers[0].vars["bias"], g["mlp_bias"], "mlp_bias")
    close(model.node_pred_vars["weights"], head["weights"], "head")
    if d:
        close(model.embeds, demb, "embeds")
    # the transposes are cached on the model, keyed by the CSR tensors
    g0 = model._full_neighbor_graph
    assert fnt.full_neighbor_graph(model, g0.indptr, g0.indices) is g0
    g0.indptr.add_(0)                                                        # a new _version: rebuilt
    assert fnt.full_neighbor_graph(model, g0.indptr, g0.indices) is not g0


@pytest.mark.parametrize("kind", ["mean", "gcn", "maxpool", "meanpool"])
def test_inference_is_the_training_forward_and_leaves_the_cache_alone(cpu_kernels, kind):
    r = np.random.RandomState(12)
    indptr, indices = messy_graph(seed=6)
    N, F = len(indptr) - 1, 6
    feats = np.vstack([r.randn(N, F).astype(np.float32), np.zeros((1, F), np.float32)])
    infos = [gs.SAGEInfo("node", None, 3, 8), gs.SAGEInfo("node", None, 3, 8)]
    model = SupervisedGraphsage(3, {}, torch.from_numpy(feats), torch.zeros((N + 1, 3), dtype=torch.int32), None, infos,
                                concat=kind != "gcn", aggregator_type=kind, device="cpu")
    model.aggregator_type = kind
    for a in model.aggregators:
        a.math = ops.MATH_FP32_SIMT
    node_ids = np.array([1, 4, 4, 7, 2, 20, -3, N + 5], np.int64)          # duplicates, an empty row, out of range
    emb = model.full_neighbor_embeddings(indptr, indices, node_ids)
    ref = fn.full_neighbor_embeddings(feats, indptr, indices, oracle_dicts(model), kind != "gcn", node_ids)
    assert emb.shape == ref.shape and np.abs(_np(emb) - ref).max() <= 1e-5
    assert not hasattr(model, "_full_neighbor_graph")                        # inference caches no transposes
    out = model.full_neighbor_outputs(indptr, indices, node_ids)
    g0 = model._full_neighbor_graph
    assert torch.equal(emb, out.detach())
    assert torch.equal(model.full_neighbor_embeddings(indptr, indices, node_ids), emb)
    assert model._full_neighbor_graph is g0                                  # nor evicts the training CSR's
