"""GPU: training step with the pooling aggregators (SURVEY 8f row 1) - loss and gradients of SupervisedGraphsage
(aggregator_type maxpool / meanpool, unfused fp32 kernels) against torch-CPU autograd on the oracle's op sequence.

A regression fails the suite."""
import numpy as np
import pytest
import torch

from conftest import load_golden, rel_err
from oracle import torch_ref

pytestmark = pytest.mark.gpu


def _cpu_outputs(adj, feats, seeds, fan, aggs, concat, pool, seed, counter):
    adj_t, feats_t, seeds_t = torch.from_numpy(adj), torch.from_numpy(feats), torch.from_numpy(seeds)
    L = len(fan)
    samples, support, sup = [seeds_t], [1], 1
    for k in range(L):
        t = L - k - 1
        sup *= fan[t]
        samples.append(torch_ref.sample_padded(adj_t, samples[k], fan[t], seed, counter + k).reshape(-1))
        support.append(sup)
    B = seeds_t.numel()
    hidden = [feats_t.index_select(0, s.long()) for s in samples]
    for layer in range(L):
        a, last, nxt = aggs[layer], layer == L - 1, []
        for hop in range(L - layer):
            k = fan[L - hop - 1]
            neigh, selfv = hidden[hop + 1], hidden[hop]
            n = selfv.shape[0]
            h = torch.relu(neigh @ a["mlp_weights"] + a["mlp_bias"]).reshape(n, k, -1)
            hp = h.amax(dim=1) if pool == "max" else h.mean(dim=1)
            fs, fn = selfv @ a["self_weights"], hp @ a["neigh_weights"]
            y = torch.cat([fs, fn], dim=1) if concat else fs + fn
            nxt.append(y if last else torch.relu(y))
        hidden = nxt
    out = hidden[0]
    return out / torch.sqrt(torch.clamp((out * out).sum(dim=1, keepdim=True), min=1e-12))


@pytest.mark.parametrize("kind,concat", [("maxpool", True), ("meanpool", False)])
def test_pool_loss_and_gradients_match_cpu_autograd(kind, concat):
    import graphsage_b200 as gs
    g = load_golden("khop")
    rs = np.random.RandomState(5)
    adj, feats = g["adj"], g["feats"]
    n, B, C = adj.shape[0] - 1, 16, 5
    seeds = rs.randint(0, n, size=B).astype(np.int32)
    labels = (rs.rand(B, C) < 0.3).astype(np.float32)
    fan, dim, wd = [4, 3], 8, 1e-3
    gs.set_default_math("fp32")
    sampler = gs.UniformNeighborSampler(torch.from_numpy(adj).cuda(), seed=123)
    sampler.counter = 40
    infos = [gs.SAGEInfo("node", sampler, fan[0], dim), gs.SAGEInfo("node", sampler, fan[1], dim)]
    m = gs.SupervisedGraphsage(C, {"batch_size": B, "dropout": 0.}, torch.from_numpy(feats).cuda(),
                               torch.from_numpy(adj).cuda(), None, infos, concat=concat, aggregator_type=kind,
                               sigmoid_loss=True, learning_rate=0.01, weight_decay=wd)
    for a in m.aggregators:                           # a non-zero MLP bias so its gradient path is exercised
        a.mlp_layers[0].vars["bias"].data.add_(torch.randn_like(a.mlp_layers[0].vars["bias"]) * 0.1)
    aggs = []
    for a in m.aggregators:
        d = {k: v.detach().cpu().clone().requires_grad_(True) for k, v in a.vars.items()}
        d["mlp_weights"] = a.mlp_layers[0].vars["weights"].detach().cpu().clone().requires_grad_(True)
        d["mlp_bias"] = a.mlp_layers[0].vars["bias"].detach().cpu().clone().requires_grad_(True)
        aggs.append(d)
    head = {k: v.detach().cpu().clone().requires_grad_(True) for k, v in m.node_pred_vars.items()}
    out = _cpu_outputs(adj, feats, seeds, fan, aggs, concat, "max" if kind == "maxpool" else "mean", 123, 40)
    logits = out @ head["weights"] + head["bias"]
    ref = torch.nn.functional.binary_cross_entropy_with_logits(logits, torch.from_numpy(labels))
    for a in aggs:                                    # the reference decays aggregator.vars only, not the Dense variables
        for k in ("neigh_weights", "self_weights"):
            ref = ref + wd * 0.5 * (a[k] * a[k]).sum()
    for v in head.values():
        ref = ref + wd * 0.5 * (v * v).sum()
    ref.backward()
    loss = m.loss(torch.from_numpy(seeds), torch.from_numpy(labels))
    loss.backward()
    assert abs(float(loss) - float(ref)) < 1e-5 * max(1.0, abs(float(ref)))
    for a, ra in zip(m.aggregators, aggs):
        for k in a.vars:
            assert rel_err(a.vars[k].grad.cpu().numpy(), ra[k].grad.numpy(), floor=1e-8) < 2e-4, (kind, k)
        assert rel_err(a.mlp_layers[0].vars["weights"].grad.cpu().numpy(), ra["mlp_weights"].grad.numpy(), floor=1e-8) < 2e-4
        assert rel_err(a.mlp_layers[0].vars["bias"].grad.cpu().numpy().reshape(1, -1),
                       ra["mlp_bias"].grad.numpy().reshape(1, -1), floor=1e-8) < 2e-4
    m.train_step(torch.from_numpy(seeds), torch.from_numpy(labels))      # clipped Adam over all variables incl. the MLP's


def test_maxpool_fp32_arithmetic_over_a_bf16_table():
    """A bf16 feature table with fp32 arithmetic takes the materialised pooling path (rows widened to fp32 by
    gs_gather_rows_f32): same answer as the fp32 table holding the bf16-rounded values (reference aggregators.py:168-195)."""
    import graphsage_b200 as gs
    from conftest import bf16_round
    g = load_golden("khop")
    rs = np.random.RandomState(8)
    n, f, B = 300, 50, 48
    adj = np.ascontiguousarray(g["adj"][:, :32])
    feats = bf16_round(np.vstack([rs.randn(n, f).astype(np.float32), np.zeros((1, f), np.float32)]))
    seeds = rs.randint(0, n, size=B).astype(np.int32)
    outs = []
    gs.set_default_math("fp32")
    for table in (torch.from_numpy(feats).cuda(), torch.from_numpy(feats).cuda().to(torch.bfloat16)):
        gs.inits.manual_seed(11)
        sampler = gs.UniformNeighborSampler(torch.from_numpy(adj).cuda(), seed=5)
        infos = [gs.SAGEInfo("node", sampler, 25, 64), gs.SAGEInfo("node", sampler, 10, 64)]
        m = gs.SampleAndAggregate({"batch_size": B, "dropout": 0.}, table, torch.from_numpy(adj).cuda(), None, infos,
                                  concat=True, aggregator_type="maxpool")
        outs.append(m.forward(torch.from_numpy(seeds), normalize=True).cpu().numpy())
    assert rel_err(outs[1], outs[0]) < 1e-6
