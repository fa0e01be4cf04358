"""CPU: training dropout over sampled blocks.  The oracle (oracle/sampled_blocks_dropout.py): its per-entry offsets
against a scalar Floyd restatement, its masked forward and gradients against float64 autograd of a dense per-edge-mask
restatement over S_l, and its equality with the masked whole-neighbourhood minibatch when every fanout covers every row.
Then the model's autograd wiring with the oracle standing in for the kernels, the refusals and the counters."""
import numpy as np
import pytest
import torch

import oracle.full_neighbor_dropout as fd
import oracle.sampled_blocks as sb
import oracle.sampled_blocks_dropout as sbd
from graphsage_b200 import full_neighbor_training as fnt
from graphsage_b200 import ops
from graphsage_b200.supervised_models import SupervisedGraphsage, full_neighbor_site_plan
from graphsage_b200.unsupervised_models import UnsupervisedGraphsage
from oracle.dropout import keep_mask, keep_prob
from oracle.full_neighbor_blocks import clamp_ids
from oracle.numerics import gather_clamped
from oracle.philox import philox4x32_10, split64
import test_full_neighbor_dropout_cpu as fdt
from test_full_neighbor_dropout_cpu import _agg_dicts, _model, messy_graph, oracle_dicts
from test_full_neighbor_minibatch_cpu import _FakeNegatives, _FakeTableRows, _fake_sage_gemm
from test_sampled_blocks_cpu import _sampled_bare, _with_sampler, rows_graph

_np = fdt._np
CSR = fdt.CSR


def scalar_offsets(indptr, v, k, seed, call, layer):
    """The raw-row offsets of S_layer(v), one Floyd move at a time from the contract's words."""
    d = max(int(indptr[v + 1]) - int(indptr[v]), 0)
    if d <= k:
        return list(range(d))
    k0, k1 = split64(seed)
    taken = []
    for i in range(k):
        u = int(philox4x32_10(np.array([i, v, call & 0xFFFFFFFF, 0x70000000 | layer], np.uint32),
                              np.array([k0, k1], np.uint32))[0])
        j = d - k + i
        t = (u * (j + 1)) >> 32
        taken.append(j if t in taken else t)
    return sorted(taken)


# ---------------------------------------------------------------- the offsets
@pytest.mark.parametrize("k", [1, 3, 10, 256])
def test_offsets_equal_the_scalar_restatement(k):
    # d <= k, d = k + 1, hubs, empty rows; duplicates, self loops and out-of-range entries (rows_graph)
    degrees = [0, 1, k, k + 1, 2 * k + 3, 0, 300, 5, k + 1, 600, 0, 2]
    indptr, indices = rows_graph(degrees, seed=k)
    N = len(indptr) - 1
    o_ptr, o = sbd.sample_offsets(indptr, k, 77, 3, 1)
    for v in range(N):
        assert list(o[o_ptr[v]:o_ptr[v + 1]]) == scalar_offsets(indptr, v, k, 77, 3, 1), v
    # the offsets name the sampled entries: S_l(v)'s values are indices[indptr[v] + q]
    s_ptr, s_idx = sb.sample_rows(indptr, indices, k, 77, 3, 1)
    assert np.array_equal(s_ptr, o_ptr)
    assert np.array_equal(s_idx, indices[np.repeat(indptr[:-1], np.diff(o_ptr)) + o])


@pytest.mark.parametrize("fanouts", [[1], [3, 2], [2, 256, 4]])
def test_block_offsets_align_with_the_block_entries(fanouts):
    indptr, indices = messy_graph(N=30, seed=4)
    N = len(indptr) - 1
    seeds = np.array([3, 0, 29, 29, 11, -4, N + 2, 7])
    blocks, offsets = sbd.entry_offsets(indptr, indices, seeds, fanouts, 12, 5)
    for l, (b, off) in enumerate(zip(blocks, offsets)):
        assert len(off) == len(b["indices"])
        for r in range(len(b["src_ids"]) - 1):
            lo, hi = b["indptr"][r], b["indptr"][r + 1] if r + 1 < len(b["indptr"]) else len(b["indices"])
            if hi == lo:
                continue
            v = int(b["src_ids"][r])
            q = off[lo:hi]
            assert list(q) == scalar_offsets(indptr, v, fanouts[l], 12, 5, l)
            # the block entry is the clamped raw entry, relabelled into V_l
            raw = clamp_ids(indices[indptr[v] + q], N)
            assert np.array_equal(b["src_ids"][b["indices"][lo:hi]], raw)


def test_slots_map_to_offsets():
    indptr, indices = messy_graph(N=20, seed=2)
    blocks, offsets = sbd.entry_offsets(indptr, indices, [1, 5, 19], [2, 2], 3, 0)
    b, off = blocks[0], offsets[0]
    t_ptr, t_idx, t_slot = fd.csr_transpose_slots(b["indptr"], b["indices"], True)
    got = sbd.slots_to_offsets(t_slot, t_idx, b["indptr"], off)
    assert np.array_equal(got < 0, t_slot < 0) and np.array_equal(got[t_slot < 0], t_slot[t_slot < 0])
    s = t_slot >= 0
    assert np.array_equal(got[s], off[b["indptr"][t_idx[s]] + t_slot[s]])


# ---------------------------------------------------------------- the masked forward and gradients
def _torch_formula(feats, indptr, indices, aggs, concat, node_ids, pw, pb, labels, sites, d, fanouts, seed, call):
    """The masked loss in float64 torch over S_l (every node sampled at layer l) with explicit per-edge mask tensors:
    edge j of v at indptr[v] + q_j, an empty row's dummy edge at nnz + v, node masks by id, the head by row."""
    N, nnz = len(indptr) - 1, len(indices)

    def edges(l):
        s_ptr, s_idx = sb.sample_rows(indptr, indices, fanouts[l], seed, call, l)
        o_ptr, o = sbd.sample_offsets(indptr, fanouts[l], seed, call, l)
        dst, src, pos = [], [], []
        for v in range(N + 1):
            c = s_ptr[v + 1] - s_ptr[v] if v < N else 0
            if c > 0:
                e = s_idx[s_ptr[v]:s_ptr[v + 1]]
                dst += [v] * c
                src += list(np.where((e < 0) | (e > N), N, e))
                pos += list(indptr[v] + o[o_ptr[v]:o_ptr[v + 1]])
            else:
                dst, src, pos = dst + [v], src + [N], pos + [nnz + v]
        return (torch.tensor(np.array(a, np.int64)) for a in (dst, src, pos))

    def mask(site, p, F):
        return torch.from_numpy(keep_mask(*site, np.asarray(p), F).astype(np.float64)) / float(keep_prob(site[2]))

    emb = torch.from_numpy(feats[:, :d].astype(np.float64)).requires_grad_(True) if d else None
    h = torch.from_numpy(feats.astype(np.float64))
    if d:
        h = torch.cat([emb, h[:, d:]], dim=1)
    params = [{k: torch.from_numpy(v.astype(np.float64)).requires_grad_(True) for k, v in a.items() if k != "type"}
              for a in aggs]
    ids = torch.from_numpy(clamp_ids(node_ids, N).astype(np.int64))
    nodes = torch.arange(N + 1)
    for l, (a, p) in enumerate(zip(aggs, params)):
        dst, src, pos = edges(l)
        cnt = torch.bincount(dst, minlength=N + 1).to(torch.float64).unsqueeze(1)
        last = l == len(aggs) - 1
        F = h.shape[1]
        if a["type"] in ("mean", "gcn"):
            s = torch.zeros_like(h).index_add(0, dst, h[src] * mask(sites[(l, "neigh")], pos, F))
            if a["type"] == "gcn":
                y = ((s + h * mask(sites[(l, "self")], nodes, F)) / (cnt + 1)) @ p["weights"]
            else:
                fs = (h * mask(sites[(l, "self")], nodes, F)) @ p["self_weights"]
                fn_ = (s / cnt) @ p["neigh_weights"]
                y = torch.cat([fs, fn_], 1) if concat else fs + fn_
        else:
            z = torch.relu((h * mask(sites[(l, "mlp")], nodes, F)) @ p["mlp_weights"] + p["mlp_bias"])
            if a["type"] == "maxpool":
                nb = torch.zeros_like(z).scatter_reduce(0, dst.unsqueeze(1).expand(-1, z.shape[1]), z[src], "amax",
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
    loss = loss + 0.01 * 0.5 * sum((v * v).sum() for v in decayed)
    loss.backward()
    return float(loss.detach()), [{k: v.grad.numpy() for k, v in p.items()} for p in params], \
        {"weights": W.grad.numpy(), "bias": b.grad.numpy()}, (emb.grad.numpy() if d else None)


@pytest.mark.parametrize("kind", ["mean", "gcn", "maxpool", "meanpool"])
@pytest.mark.parametrize("concat", [True, False])
@pytest.mark.parametrize("d,fanouts", [(0, [2]), (16, [3, 2]), (0, [1, 4, 2])])
def test_oracle_gradients_equal_float64_autograd_over_the_sample(kind, concat, d, fanouts):
    r = np.random.RandomState(8)
    indptr, indices = messy_graph(seed=9)
    N, F, C, L = len(indptr) - 1, 5, 3, len(fanouts)
    x = r.randint(0, 3, size=(N + 1, F)).astype(np.float32) if kind == "maxpool" else r.randn(N + 1, F).astype(np.float32)
    x[N] = 0
    feats = np.concatenate([r.randn(N + 1, d).astype(np.float32), x], 1) if d else x
    aggs = _agg_dicts(kind, [d + F] + [4] * L, concat, r)
    node_ids = np.array([0, 3, 5, 5, 9, 2, 23, 3, -1], np.int64)
    out_w = 4 * (2 if concat and kind != "gcn" else 1)
    pw, pb = (r.randn(out_w, C) * 0.5).astype(np.float32), (r.randn(C) * 0.1).astype(np.float32)
    labels = np.eye(C)[r.randint(0, C, len(node_ids))]
    sites = fd.sites(kind, L, True, 31, 7, 0.5)
    loss, grads, head, demb = sbd.sampled_loss_grads_dropout(feats, indptr, indices, aggs, concat, node_ids, labels, pw,
                                                             pb, fanouts, 6, 2, sites, False, 0.01, d)
    rl, rg, rh, rd = _torch_formula(feats, indptr, indices, aggs, concat, node_ids, pw, pb, labels, sites, d, fanouts,
                                    6, 2)
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


@pytest.mark.parametrize("kind", ["mean", "gcn", "maxpool", "meanpool"])
@pytest.mark.parametrize("L", [1, 2, 3])
def test_large_fanouts_mask_as_the_whole_neighbourhood_blocks(kind, L):
    indptr, indices = messy_graph(seed=7)
    N = len(indptr) - 1
    r = np.random.RandomState(3)
    feats = np.vstack([r.randn(N, 5).astype(np.float32), np.zeros((1, 5), np.float32)])
    concat = kind != "gcn"
    aggs = _agg_dicts(kind, [5] + [4] * L, concat, r)
    seeds = np.array([3, 0, 23, 23, 11, -4, N + 2])
    sites = fd.sites(kind, L, False, 99, 40, 0.4)
    fan = [int(np.diff(indptr).max())] * L
    got = sbd.sampled_block_outputs(feats, indptr, indices, aggs, concat, seeds, fan, 5, 1, sites)
    assert np.array_equal(got, fd.block_outputs(feats, indptr, indices, aggs, concat, seeds, sites))
    small = sbd.sampled_block_outputs(feats, indptr, indices, aggs, concat, seeds, [2] * L, 5, 1, sites)
    assert not np.array_equal(got, small)


def test_a_node_masks_its_layer0_sum_alike_in_every_batch():
    indptr, indices = messy_graph(N=30, seed=3)
    N = len(indptr) - 1
    r = np.random.RandomState(1)
    feats = np.vstack([r.randn(N, 6).astype(np.float32), np.zeros((1, 6), np.float32)])
    rows = {}
    for seeds in ([4, 9], [4, 17, 22, 9], [1, 2, 3, 4]):
        blocks, offsets = sbd.entry_offsets(indptr, indices, seeds, [3], 8, 0)
        b = blocks[0]
        m = sbd.csr_aggregate_dropout_offsets(gather_clamped(feats, b["src_ids"]), b["indptr"], b["indices"], "mean",
                                              (2, 5, 0.5), (2, 6, 0.5), (indptr, b["src_ids"], len(indices), offsets[0]),
                                              b["rows"])
        for i, s in enumerate(clamp_ids(seeds, N)):
            rows.setdefault(int(s), []).append(m[i])
    assert all(np.array_equal(a[0], x) for a in rows.values() for x in a) and len(rows[4]) == 3


# ---------------------------------------------------------------- the autograd wiring, kernels replaced by the oracle
def _fake_csr_aggregate(src, indptr, indices, op, rows=None, out=None, dropout=None, t_slot=None):
    if dropout is not None and len(dropout[2]) == 4:
        ns, ss, pm = dropout
        return torch.from_numpy(sbd.csr_aggregate_dropout_offsets(
            _np(src), _np(indptr), _np(indices), op, ns[:3], ss[:3], (*fdt._pm(pm[:3]), _np(pm[3])),
            None if rows is None else _np(rows)))
    return fdt._fake_csr_aggregate(src, indptr, indices, op, rows, out, dropout, t_slot)


def _fake_blocks(indptr, indices, seeds, n_layers, fanouts=None, seed=0, call=0, entry_offsets=False):
    assert fanouts is not None and len(fanouts) == n_layers
    blocks, offsets = sbd.entry_offsets(_np(indptr), _np(indices), _np(seeds), fanouts, seed, call)
    out = [ops.CsrBlock(*(torch.from_numpy(np.asarray(b[k])) for k in ("src_ids", "indptr", "indices", "rows")))
           for b in blocks]
    _fake_blocks.calls.append(entry_offsets)
    return (out, [torch.from_numpy(o.astype(np.int32)) for o in offsets]) if entry_offsets else out


@pytest.fixture()
def kernels(fdt_kernels, monkeypatch):
    _fake_blocks.calls = []
    monkeypatch.setattr(ops, "csr_aggregate", _fake_csr_aggregate)
    monkeypatch.setattr(ops, "csr_blocks", _fake_blocks)
    monkeypatch.setattr(ops, "csr_slots_to_offsets", lambda t_slot, t_indices, indptr, pos_off: torch.from_numpy(
        sbd.slots_to_offsets(_np(t_slot), _np(t_indices), _np(indptr), _np(pos_off)).astype(np.int32)))
    monkeypatch.setattr(ops, "sage_gemm", _fake_sage_gemm)
    monkeypatch.setattr(ops, "TableRows", _FakeTableRows)
    monkeypatch.setattr(ops, "gather_rows_f32", lambda feats, ids=None, row0=0, n=None, out=None:
                        feats[ids.long()].float().clone())


@pytest.fixture()
def fdt_kernels(monkeypatch):
    monkeypatch.setattr(ops, "csr_transpose", fdt._fake_transpose)
    monkeypatch.setattr(ops, "csr_max_backward", fdt._fake_max_backward)
    monkeypatch.setattr(ops, "embedding_grad", fdt._fake_embedding_grad)
    monkeypatch.setattr(ops, "dropout_apply", fdt._fake_dropout_apply)
    monkeypatch.setattr(ops, "l2_normalize_rows_", fdt._fake_l2_)
    monkeypatch.setattr(ops, "gather_rows", lambda src, ids, out=None: src[ids.long()].clone())
    monkeypatch.setattr(torch.cuda, "is_current_stream_capturing", lambda: False)


@pytest.mark.parametrize("kind,concat,d", [("mean", True, 0), ("gcn", False, 16), ("maxpool", True, 16),
                                           ("meanpool", False, 0), ("mean", False, 16)])
def test_supervised_wiring_matches_the_oracle(kernels, kind, concat, d):
    r = np.random.RandomState(11)
    indptr, indices = messy_graph(seed=5)
    N, C = len(indptr) - 1, 3
    model = _model(kind, concat, d, N, 6, r, rate=0.5)
    sampler = _with_sampler(model, seed=5, counter=3)
    model.dropout_counter = 9
    node_ids = np.array([1, 4, 4, 7, 2, 20, -3], np.int64)
    labels = np.eye(C)[r.randint(0, C, len(node_ids))]
    loss = model.sampled_minibatch_loss(indptr, indices, node_ids, labels, dropout=model.dropout_rate)
    assert model.dropout_counter == 9 + len(full_neighbor_site_plan(kind, 2, head=True)) and sampler.counter == 4
    assert _fake_blocks.calls == [True]
    loss.backward()
    fanouts = [info.num_samples for info in model.layer_infos]
    rl, grads, head, demb = sbd.sampled_loss_grads_dropout(
        _np(model.features), indptr, indices, oracle_dicts(model), concat, node_ids, labels,
        _np(model.node_pred_vars["weights"]), _np(model.node_pred_vars["bias"]), fanouts, 5, 3,
        fd.sites(kind, 2, True, 77, 9, 0.5), False, 0.01, d)
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
    # inference never drops, and leaves the dropout counter alone
    with torch.no_grad():
        emb = model.sampled_minibatch_embeddings(indptr, indices, node_ids)
    want = sb.sampled_embeddings(_np(model.features), indptr, indices, oracle_dicts(model), concat, node_ids, fanouts,
                                 5, 4)
    assert np.abs(_np(emb) - want).max() < 1e-5 and sampler.counter == 5
    assert model.dropout_counter == 9 + len(full_neighbor_site_plan(kind, 2, head=True))


@pytest.mark.parametrize("kind", ["mean", "gcn", "maxpool"])
def test_rate_zero_is_dropout_none(kernels, kind):
    r = np.random.RandomState(12)
    indptr, indices = messy_graph(seed=6)
    model = _model(kind, kind != "gcn", 0, len(indptr) - 1, 6, r)
    sampler = _with_sampler(model, seed=2, counter=0)
    ids = np.array([1, 4, 4, 7, 2, 20])
    a = model.sampled_minibatch_outputs(indptr, indices, ids)
    sampler.counter = 0
    b = model.sampled_minibatch_outputs(indptr, indices, ids, dropout=0.)
    assert torch.equal(a, b) and model.dropout_counter == 0 and _fake_blocks.calls == [False, False]
    sampler.counter = 0
    c = model.sampled_minibatch_outputs(indptr, indices, ids, dropout=0.5)
    assert not torch.equal(a, c) and model.dropout_counter == len(full_neighbor_site_plan(kind, 2))
    assert _fake_blocks.calls[-1] is True and sampler.counter == 1


def test_unsupervised_wiring(kernels):
    r = np.random.RandomState(13)
    indptr, indices = messy_graph(seed=8)
    N = len(indptr) - 1
    feats = np.vstack([r.randn(N, 6).astype(np.float32), np.zeros((1, 6), np.float32)])
    import graphsage_b200 as gs
    infos = [gs.SAGEInfo("node", None, 3, 8), gs.SAGEInfo("node", None, 2, 8)]
    model = UnsupervisedGraphsage({"dropout": 0.3}, torch.from_numpy(feats), torch.zeros((N + 1, 3), dtype=torch.int32),
                                  np.ones(N + 1), infos, concat=True, aggregator_type="mean", weight_decay=0.01,
                                  device="cpu", neg_sample_size=4, dropout_seed=4)
    model.aggregator_type = "mean"
    for a in model.aggregators:
        a.math = ops.MATH_FP32_SIMT
    sampler = _with_sampler(model, seed=9, counter=0)
    model.neg_sampler = _FakeNegatives([5, 0, 23, 5])
    b1, b2 = np.array([1, 2, 3, 9]), np.array([4, 4, 20, 0])
    loss = model.sampled_minibatch_loss(indptr, indices, b1, b2, dropout=model.dropout_rate)
    assert model.neg_sampler.counter == 1 and sampler.counter == 1 and model.dropout_counter == 4
    loss.backward()
    # the same loss from one masked block set over cat(b1, b2, neg) at sampler call 0 and dropout call 0
    sampler.counter, model.dropout_counter = 0, 0
    out = fnt.full_neighbor_outputs(model, indptr, indices, torch.cat([torch.tensor(b1), torch.tensor(b2),
                                                                       model.neg_sampler.ids.long()]),
                                    minibatch=True, sampled=True, dropout=0.3)
    assert torch.equal(loss.detach(), model._pairs_loss(*torch.split(out, [4, 4, 4])).detach())
    want = sbd.sampled_block_outputs(feats, indptr, indices, oracle_dicts(model), True,
                                     np.concatenate([b1, b2, _np(model.neg_sampler.ids)]), [3, 2], 9, 0,
                                     fd.sites("mean", 2, False, 4, 0, 0.3))
    assert np.abs(_np(out) - want).max() < 1e-5
    model.sampled_minibatch_train_step(indptr, indices, b1, b2, dropout=0.3)
    assert model.neg_sampler.counter == 2 and sampler.counter == 2 and model.dropout_counter == 8


# ---------------------------------------------------------------- refusals and counters (no GPU needed: they fire first)
def test_refusals_draw_nothing():
    m = _sampled_bare(dropout_rate=0.5)
    m.dropout_counter = 0
    with pytest.raises(NotImplementedError, match="dropout"):
        m.sampled_minibatch_loss(*CSR, [0], [[1.0]])
    with pytest.raises(NotImplementedError, match="dropout"):
        m.sampled_minibatch_outputs(*CSR, [0], dropout=None)
    for bad in (-0.1, 1.0, float("nan"), "0.5", True):
        with pytest.raises(ValueError, match="dropout"):
            m.sampled_minibatch_train_step(*CSR, [0], [[1.0]], dropout=bad)
    with pytest.raises(NotImplementedError, match="distributed"):
        _sampled_bare(distributed=True, dropout_rate=0.5).sampled_minibatch_loss(*CSR, [0], [[1.0]], dropout=0.5)
    with pytest.raises(NotImplementedError, match="seq"):
        _sampled_bare("seq").sampled_minibatch_outputs(*CSR, [0], dropout=0.5)
    assert m.layer_infos[0].neigh_sampler.counter == 0 and m.dropout_counter == 0
    u = UnsupervisedGraphsage.__new__(UnsupervisedGraphsage)
    u.__dict__.update(_sampled_bare(dropout_rate=0.1).__dict__)
    u.neg_sampler = _FakeNegatives([0])
    with pytest.raises(NotImplementedError, match="dropout"):
        u.sampled_minibatch_loss(*CSR, [0], [1])
    with pytest.raises(ValueError, match="dropout"):
        u.sampled_minibatch_loss(*CSR, [0], [1], dropout=2.)
    u.distributed = True
    with pytest.raises(NotImplementedError, match="distributed"):
        u.sampled_minibatch_loss(*CSR, [0], [1], dropout=0.1)
    assert u.neg_sampler.counter == 0 and u.layer_infos[0].neigh_sampler.counter == 0


def test_ops_refuse_bad_offsets():
    with pytest.raises(ValueError, match="entry_offsets"):
        ops.csr_blocks(torch.zeros(3, dtype=torch.int64), torch.zeros(0, dtype=torch.int32),
                       torch.zeros(1, dtype=torch.int32), 1, entry_offsets=True)
    with pytest.raises(RuntimeError, match="CUDA-only"):
        ops.csr_slots_to_offsets(*(torch.zeros(2, dtype=torch.int32),) * 2, torch.zeros(3, dtype=torch.int64),
                                 torch.zeros(2, dtype=torch.int32))
