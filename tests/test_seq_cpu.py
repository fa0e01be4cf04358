"""The LSTM sequence aggregator (graphsage_seq) without a GPU: the oracle against the fixture made by the reference's own
SeqAggregator (tests/golden/seq.npz), the oracle's BPTT against fp64 autograd, the dropout site plan, the parameter lists,
the refusals, and the autograd wiring of _SeqAggregateRowsFn with torch stand-ins for the kernels (TEST mocks only - the
product has no such path)."""
import os

import numpy as np
import pytest
import torch

import graphsage_b200 as gs
from graphsage_b200 import ops, supervised_models as sm
from oracle import seq as oseq
from oracle.aggregate import identity, relu

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "seq.npz")


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


def test_length_rule_counts_rows_with_a_nonzero_element():
    x = np.ones((5, 4, 3), np.float32)
    x[1, 1] = 0.0                 # interspersed: still counted by position, len = 3
    x[2] = 0.0                    # all zero: clamped to 1
    x[3, 0] = -0.0                # negative zeros are zero
    x[4, :, 1:] = 0.0             # one non-zero element is enough
    assert oseq.seq_lengths(x).tolist() == [4, 3, 1, 3, 4]


def _kernel(g, prefix):
    """The cell kernel the fixture was written with: it stores the seed and shape (oracle.seq.cell_kernel)."""
    return oseq.cell_kernel(g[prefix + "_kernel_seed"], g[prefix + "_kernel_shape"])


@pytest.mark.parametrize("tag", ["c0", "c1", "bias", "big"])
def test_oracle_matches_the_reference_aggregator(golden, tag):
    g = golden
    concat = tag in ("c1", "big")
    kernel = _kernel(g, tag)
    got = oseq.seq_aggregator(g["self"], g["neigh"], kernel, g[tag + "_cell_bias"], g[tag + "_nw"],
                              g[tag + "_sw"], concat=concat, act=relu, bias=g[tag + "_bias"] if tag == "bias" else None)
    np.testing.assert_allclose(got, g[tag + "_out"], rtol=1e-5, atol=1e-6)
    assert int(g[tag + "_dropout_calls"]) == 0            # built with dropout=0.5: the aggregator draws no mask
    H = 256 if tag == "big" else 128
    assert kernel.shape == (g["neigh"].shape[2] + H, 4 * H) and g[tag + "_nw"].shape[0] == H


def test_oracle_khop_matches_the_reference_aggregate(golden):
    g = golden
    fan, support = [int(v) for v in g["khop_fanout"]], [int(v) for v in g["khop_support"]]
    samples = [g["khop_samples%d" % h] for h in range(len(fan) + 1)]
    aggs = [dict(kernel=_kernel(g, "khop_L%d" % li), cell_bias=g["khop_L%d_cell_bias" % li], neigh_weights=g["khop_L%d_nw" % li],
                 self_weights=g["khop_L%d_sw" % li]) for li in range(len(fan))]
    got = oseq.aggregate_khop_seq(samples, g["khop_feats"], fan, support, len(g["khop_seeds"]), aggs, True)
    np.testing.assert_allclose(got, g["khop_out"], rtol=1e-5, atol=1e-6)


def test_oracle_bptt_matches_fp64_autograd():
    r = np.random.RandomState(5)
    n, k, H = 6, 5, 8
    P = r.randn(n, k, 4 * H)
    Wh = r.randn(H, 4 * H) * 0.3
    lengths = np.array([5, 1, 3, 2, 5, 4], np.int32)
    h, gates, cs, hp = oseq.lstm_run(P, Wh, lengths, train=True, dtype=np.float64)
    R = r.randn(n, H)
    dZ = oseq.lstm_bptt(R, gates, cs, lengths, Wh)
    Pt = torch.from_numpy(P).requires_grad_(True)
    Wt = torch.from_numpy(Wh)
    ht, ct = torch.zeros(n, H, dtype=torch.float64), torch.zeros(n, H, dtype=torch.float64)
    L = torch.from_numpy(lengths)
    for t in range(k):
        on = (t < L).unsqueeze(1)
        z = Pt[:, t] + ht @ Wt
        cn = ct * torch.sigmoid(z[:, 2 * H:3 * H] + 1.0) + torch.sigmoid(z[:, :H]) * torch.tanh(z[:, H:2 * H])
        hn = torch.tanh(cn) * torch.sigmoid(z[:, 3 * H:])
        ct, ht = torch.where(on, cn, ct), torch.where(on, hn, ht)
    np.testing.assert_allclose(ht.detach().numpy(), h, rtol=1e-12, atol=1e-12)
    (ht * torch.from_numpy(R)).sum().backward()
    np.testing.assert_allclose(dZ, Pt.grad.numpy(), rtol=1e-10, atol=1e-12)
    # h_prev and the weight gradient dW_h = sum_t h_{t-1}^T dz_t
    Wt2 = torch.from_numpy(Wh).requires_grad_(True)
    ht, ct = torch.zeros(n, H, dtype=torch.float64), torch.zeros(n, H, dtype=torch.float64)
    for t in range(k):
        on = (t < L).unsqueeze(1)
        z = torch.from_numpy(P[:, t]) + ht @ Wt2
        cn = ct * torch.sigmoid(z[:, 2 * H:3 * H] + 1.0) + torch.sigmoid(z[:, :H]) * torch.tanh(z[:, H:2 * H])
        hn = torch.tanh(cn) * torch.sigmoid(z[:, 3 * H:])
        ct, ht = torch.where(on, cn, ct), torch.where(on, hn, ht)
    (ht * torch.from_numpy(R)).sum().backward()
    np.testing.assert_allclose(hp.reshape(n * k, H).T @ dZ.reshape(n * k, 4 * H), Wt2.grad.numpy(), rtol=1e-10, atol=1e-12)


def test_site_plan_has_no_aggregator_sites_for_seq():
    assert sm.dropout_site_plan("seq", 2) == []
    assert sm.dropout_site_plan("seq", 3, head=True) == [(None, None, "head")]
    assert len(sm.dropout_site_plan("mean", 2)) == 6                 # unchanged for the other kinds


def test_hidden_widths_and_parameter_lists():
    for size, H in (("small", 128), ("big", 256)):
        a = gs.SeqAggregator(10, 4, model_size=size, neigh_input_dim=12, concat=True, bias=True, device="cpu")
        assert a.hidden_dim == H and tuple(a.cell.vars["kernel"].shape) == (12 + H, 4 * H)
        assert tuple(a.cell.vars["bias"].shape) == (4 * H,) and not a.cell.vars["bias"].any()
        assert tuple(a.vars["neigh_weights"].shape) == (H, 4) and tuple(a.vars["self_weights"].shape) == (10, 4)
        assert tuple(a.vars["bias"].shape) == (8,)
        assert a.cell.W_x.data_ptr() == a.cell.vars["kernel"].data_ptr() and tuple(a.cell.W_h.shape) == (H, 4 * H)
    with pytest.raises(ValueError):
        gs.SeqAggregator(10, 4, model_size="huge", device="cpu")
    s = gs.SeqAggregator(8, 4, device="cpu")
    m = gs.MaxPoolingAggregator(8, 4, device="cpu")
    every, decayed = sm.aggregator_parameters([s, m])
    ids = {id(t) for t in decayed}
    assert len(decayed) == 4 and len(every) == 4 + 2 + 2
    assert id(s.cell.vars["kernel"]) not in ids and id(s.cell.vars["bias"]) not in ids
    assert every[-2:] == [s.cell.vars["kernel"], s.cell.vars["bias"]]
    g = gs.MeanAggregator(8, 4, device="cpu")
    assert sm.aggregator_parameters([g, m])[0] == list(g.vars.values()) + list(m.vars.values()) + \
        list(m.mlp_layers[0].vars.values())


def _model_args(features, n=30):
    adj = torch.zeros((n + 1, 4), dtype=torch.int32)
    sampler = object()                                   # never called: the constructors only
    infos = [gs.SAGEInfo("node", sampler, 3, 8), gs.SAGEInfo("node", sampler, 2, 8)]
    return ({"batch_size": 4, "dropout": 0.}, features, adj, np.ones(n + 1), infos)


def test_refusals():
    f = torch.zeros((31, 6), dtype=torch.float32)
    with pytest.raises(NotImplementedError, match="bfloat16"):
        gs.SupervisedGraphsage(3, *_model_args(f.to(torch.bfloat16)), aggregator_type="seq", device="cpu")
    with pytest.raises(NotImplementedError, match="bfloat16"):
        gs.SampleAndAggregate(*_model_args(f.to(torch.bfloat16)), aggregator_type="seq", device="cpu")
    with pytest.raises(NotImplementedError, match="fused_pool"):
        gs.SupervisedGraphsage(3, *_model_args(f), aggregator_type="seq", device="cpu", fused_pool=True)
    with pytest.raises(NotImplementedError, match="fused_pool"):
        gs.UnsupervisedGraphsage(*_model_args(f), aggregator_type="seq", device="cpu", fused_pool=True)

    class Sharded(object):
        c_table = None
        dtype = torch.float32
        shape = (31, 6)
    with pytest.raises(NotImplementedError, match="ShardedFeatures"):
        gs.aggregators.refuse_seq_table(Sharded())
    a = gs.SeqAggregator(6, 4, device="cpu")
    with pytest.raises(NotImplementedError, match="ShardedFeatures"):
        a.aggregate_rows(Sharded(), [ops.Seg(2, 3)])
    # accepted: both training classes, fp32 table
    m = gs.SupervisedGraphsage(3, *_model_args(f), aggregator_type="seq", device="cpu")
    assert all(isinstance(x, gs.SeqAggregator) for x in m.aggregators) and m.aggregators[0].hidden_dim == 128
    m = gs.UnsupervisedGraphsage(*_model_args(f), aggregator_type="seq", model_size="big", device="cpu")
    assert m.aggregators[1].hidden_dim == 256


# ---------------------------------------------------------------- autograd wiring with torch stand-ins for the kernels
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


def _fake_seq_lengths(x, n, k):
    return torch.from_numpy(oseq.seq_lengths(x.reshape(n, k, -1).numpy()))


def _fake_lstm_forward(P, Wh, lengths, n, k, out=None, train=False):
    h, g, c, hp = oseq.lstm_run(P.reshape(n, k, -1).numpy(), Wh.numpy(), lengths.numpy(), train=True)
    h = torch.from_numpy(h)
    if out is not None:
        out.copy_(h)
        h = out
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a.reshape(n * k, -1)))  # noqa: E731
    return (h, t(g), t(c), t(hp)) if train else h


def _fake_lstm_backward(dh_last, gates, c, lengths, Wh, n, k):
    dZ = oseq.lstm_bptt(dh_last.numpy(), gates.reshape(n, k, -1).numpy(), c.reshape(n, k, -1).numpy(), lengths.numpy(),
                        Wh.numpy(), dtype=np.float32)
    return torch.from_numpy(dZ.reshape(n * k, -1))


def _fake_embedding_grad(emb_shape, lists, sites=None):
    out = torch.zeros(emb_shape)
    for ids, g, group, scale in lists:
        rows = g.repeat_interleave(group, dim=0)[:ids.numel()] * scale
        out.index_add_(0, ids.long(), rows)
    return out


@pytest.fixture()
def cpu_kernels(monkeypatch):
    monkeypatch.setattr(sm, "_embedding_grad", _fake_embedding_grad)
    monkeypatch.setattr(ops, "sage_gemm", _fake_sage_gemm)
    monkeypatch.setattr(ops, "gather_rows", _fake_gather_rows)
    monkeypatch.setattr(ops, "seq_lengths", _fake_seq_lengths)
    monkeypatch.setattr(ops, "lstm_forward", _fake_lstm_forward)
    monkeypatch.setattr(ops, "lstm_backward", _fake_lstm_backward)


@pytest.mark.parametrize("concat", [True, False])
@pytest.mark.parametrize("identity_dim", [0, 3])
def test_two_layer_seq_chain_gradients_match_autograd(cpu_kernels, concat, identity_dim):
    r = np.random.RandomState(3)
    N, F, D, B, k1, k2 = 40, 10, 6, 5, 3, 4
    feats = torch.from_numpy(r.randn(N, F).astype(np.float32))
    feats[7] = 0.0
    s0 = torch.from_numpy(r.randint(0, N, size=B).astype(np.int32))
    s1 = torch.from_numpy(r.randint(0, N, size=B * k1).astype(np.int32))
    s2 = torch.from_numpy(r.randint(0, N, size=B * k1 * k2).astype(np.int32))
    s2[1:k2:2] = 7                                       # interspersed zero rows; with embeddings they are not zero
    s2[k2:2 * k2] = 7                                    # an all-zero sequence
    emb = None
    if identity_dim:
        emb = torch.from_numpy(r.randn(N, identity_dim).astype(np.float32)).requires_grad_(True)
    dim_mult = 2 if concat else 1
    a0 = gs.SeqAggregator(F + identity_dim, D, act=gs.relu, concat=concat, device="cpu")
    a1 = gs.SeqAggregator(dim_mult * D, D, act=gs.identity, concat=concat, device="cpu")
    params = []
    for a in (a0, a1):
        a.cell.vars["bias"] = torch.from_numpy(r.randn(a.cell.vars["bias"].numel()).astype(np.float32) * 0.1)
        for d in (a.vars, a.cell.vars):
            for key in d:
                d[key] = d[key].detach().clone().requires_grad_(True)
                params.append(d[key])

    def table():
        return torch.cat([emb, feats], dim=1) if emb is not None else feats

    seg0 = [ops.Seg(B, k1, self_ids=s0, neigh_ids=s1, out_row0=0), ops.Seg(B * k1, k2, self_ids=s1, neigh_ids=s2, out_row0=B)]
    src0 = table().detach()
    h1 = sm._SeqAggregateRowsFn.apply(a0, src0, seg0, a0.vars["self_weights"], a0.vars["neigh_weights"],
                                      a0.cell.vars["kernel"], a0.cell.vars["bias"], emb)
    seg1 = [ops.Seg(B, k1, self_row0=0, neigh_row0=B, out_row0=0)]
    out = sm._SeqAggregateRowsFn.apply(a1, h1, seg1, a1.vars["self_weights"], a1.vars["neigh_weights"],
                                       a1.cell.vars["kernel"], a1.cell.vars["bias"])
    R = torch.from_numpy(r.randn(*out.shape).astype(np.float32))
    (out * R).sum().backward()
    everything = params + ([emb] if emb is not None else [])
    got = [p.grad.clone() for p in everything]
    for p in everything:
        p.grad = None
    t = table()
    x0, x1, x2 = t[s0.long()], t[s1.long()], t[s2.long()]

    def layer(a, selfv, neigh, k, last):
        return oseq.torch_seq_layer(selfv, neigh, a.cell.vars["kernel"], a.cell.vars["bias"], a.vars["self_weights"],
                                    a.vars["neigh_weights"], k, concat, last)
    ref = layer(a1, layer(a0, x0, x1, k1, False), layer(a0, x1, x2, k2, False), k1, True)
    assert torch.allclose(out.detach(), ref.detach(), rtol=1e-5, atol=1e-5)
    (ref * R).sum().backward()
    for p, g in zip(everything, got):
        assert p.grad is not None and torch.allclose(g, p.grad, rtol=2e-4, atol=2e-5), float((g - p.grad).abs().max())
