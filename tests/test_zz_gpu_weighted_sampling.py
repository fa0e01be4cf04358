"""GPU: sampling neighbours in proportion to edge weight.  ops.sample_csr_rows(weights=) and ops.csr_blocks(
sample_weights=, entry_offsets=) byte for byte against oracle/weighted_sampling.py over toy-ppi, a graph with a
10^5-entry hub row and an edgeless graph, every weight kind, fanouts 1 .. 256 and 1 .. 4 layers; the law of the draws
on 2^20 copies of one row; the models' embeddings, losses and gradients against the oracle with and without edge_weight
and dropout; host and int8 tables; Adam steps against a CPU run; and the invariants (sample_weight=None is the uniform
path, large fanouts give the whole-neighbourhood minibatch, one counter step and one host read per block set)."""
import itertools
import warnings

import numpy as np
import pytest
import torch

from conftest import rel_err
from oracle import full_neighbor_dropout as fd
from oracle import sampled_blocks_dropout as sbd
from oracle import weighted_sampling as ws
from test_zz_gpu_full_neighbor import dev, edge_csr, oracle_aggs  # noqa: F401
from test_zz_gpu_full_neighbor_minibatch import unsup_model
from test_zz_gpu_full_neighbor_train import POOL_BIAS_TOL, named_grads, sup_model
from test_zz_gpu_sampled_blocks import _check_blocks, _set_fanouts, capped_csr, graph

pytestmark = pytest.mark.gpu
GRAD_TOL = 2e-4


@pytest.fixture(scope="module")
def gs():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    import graphsage_b200
    graphsage_b200._lib.lib()
    return graphsage_b200


def weights_of(n, kind, seed=0):
    rs = np.random.RandomState(seed)
    pos = rs.uniform(0.01, 5, n).astype(np.float32)
    if kind == "positive":
        return pos
    if kind == "equal":
        return np.full(n, 0.75, np.float32)
    if kind == "heavy":
        return np.exp(rs.randn(n) * 4).astype(np.float32)
    w = pos.copy()
    sel = rs.randint(0, 8, n)
    special = {"zeros": {0: 0.0, 1: -0.0}, "negative": {0: -1.0, 1: -3e38}, "nan": {0: np.nan},
               "inf": {0: np.inf}, "subnormal": {0: 1e-45, 1: 1e-40},
               "mixed": {0: 0.0, 1: -1.0, 2: np.nan, 3: np.inf, 4: 1e-40}}[kind]
    for s, v in special.items():
        w[sel == s] = np.float32(v)
    return w


KINDS = ["positive", "zeros", "negative", "nan", "inf", "subnormal", "equal", "heavy", "mixed"]


def _seeds(N, n=200, seed=0):
    rs = np.random.RandomState(seed)
    return np.concatenate([rs.randint(0, max(N, 1), size=n), [17, 17, -1, N, N + 4]]).astype(np.int32)


# ---------------------------------------------------------------- the kernels, bit for bit
@pytest.mark.parametrize("name", ["toy-ppi", "rmat", "messy", "empty"])
@pytest.mark.parametrize("k", [1, 10, 25, 32, 33, 256])
def test_sample_rows_bit_exact(gs, name, k):
    indptr, indices = graph(name)
    for kind in (KINDS if name != "rmat" else ["positive", "mixed", "heavy"]):
        w = weights_of(len(indices), kind, k)
        for seed, call, layer in ((123, 0, 0), (2**63 + 7, 5, 3), (0, 2**32 + 1, 7)):
            got_ptr, got_idx = gs.ops.sample_csr_rows(dev(indptr), dev(indices), k, seed, call, layer, weights=dev(w))
            want_ptr, want_idx = ws.sample_rows(indptr, indices, w, k, seed, call, layer)
            assert np.array_equal(got_ptr.cpu().numpy(), want_ptr), (kind, seed)
            assert np.array_equal(got_idx.cpu().numpy(), want_idx), (kind, seed)


@pytest.mark.parametrize("name", ["toy-ppi", "rmat", "messy", "empty"])
@pytest.mark.parametrize("k", [1, 10, 25, 32, 33, 256])
def test_weighted_blocks_and_offsets_bit_exact(gs, name, k):
    indptr, indices = graph(name)
    N = len(indptr) - 1
    seeds = _seeds(N, seed=k)
    kinds = KINDS if name in ("messy", "empty") else ["mixed", "heavy"]
    for kind, L in zip(itertools.cycle(kinds), range(1, 5)):
        w = weights_of(len(indices), kind, L)
        fanouts = [k, max(1, k // 2), k, 3][:L]
        for seed, call in ((123, 0), (2**63 + 7, 5)):
            got, offs = gs.ops.csr_blocks(dev(indptr), dev(indices), dev(seeds), L, fanouts=fanouts, seed=seed,
                                          call=call, entry_offsets=True, sample_weights=dev(w))
            blocks, want_offs = ws.entry_offsets(indptr, indices, w, seeds, fanouts, seed, call)
            _check_blocks(got, blocks)
            for o, wo in zip(offs, want_offs):
                assert o.dtype == torch.int32 and np.array_equal(o.cpu().numpy(), wo)
            plain = gs.ops.csr_blocks(dev(indptr), dev(indices), dev(seeds), L, fanouts=fanouts, seed=seed, call=call,
                                      sample_weights=dev(w))
            assert all(torch.equal(a, b) for x, y in zip(plain, got) for a, b in zip(x, y))


def test_hub_rows_spread_over_a_cta(gs):
    """Several rows of 10^5 - 10^6 entries among short ones, in one group of a CTA and across groups."""
    rs = np.random.RandomState(2)
    deg = rs.randint(0, 30, size=5000)
    deg[[3, 4, 6, 1000, 4095, 4096]] = [1000000, 100000, 4096, 4095, 250000, 5000]
    indptr = np.concatenate([[0], np.cumsum(deg)]).astype(np.int64)
    indices = rs.randint(-1, 5001, size=int(indptr[-1])).astype(np.int32)
    for kind, k in (("heavy", 25), ("mixed", 256), ("equal", 1), ("inf", 33)):
        w = weights_of(len(indices), kind, k)
        got_ptr, got_idx = gs.ops.sample_csr_rows(dev(indptr), dev(indices), k, 9, 1, 2, weights=dev(w))
        want_ptr, want_idx = ws.sample_rows(indptr, indices, w, k, 9, 1, 2)
        assert np.array_equal(got_ptr.cpu().numpy(), want_ptr) and np.array_equal(got_idx.cpu().numpy(), want_idx)
        seeds = np.array([3, 4, 6, 1000, 4095, 4096, 7, 8], np.int32)
        got, offs = gs.ops.csr_blocks(dev(indptr), dev(indices), dev(seeds), 2, fanouts=[k, k], seed=9, call=1,
                                      entry_offsets=True, sample_weights=dev(w))
        blocks, want_offs = ws.entry_offsets(indptr, indices, w, seeds, [k, k], 9, 1)
        _check_blocks(got, blocks)
        assert all(np.array_equal(o.cpu().numpy(), wo) for o, wo in zip(offs, want_offs))


def test_repeated_calls_are_byte_identical_and_a_new_call_differs(gs):
    indptr, indices = graph("rmat")
    w = dev(weights_of(len(indices), "heavy"))
    seeds = dev(_seeds(len(indptr) - 1))
    args = (dev(indptr), dev(indices), seeds, 2)
    a = gs.ops.csr_blocks(*args, fanouts=[25, 10], seed=4, call=7, entry_offsets=True, sample_weights=w)
    b = gs.ops.csr_blocks(*args, fanouts=[25, 10], seed=4, call=7, entry_offsets=True, sample_weights=w)
    c = gs.ops.csr_blocks(*args, fanouts=[25, 10], seed=4, call=8, entry_offsets=True, sample_weights=w)
    assert all(torch.equal(x, y) for bx, by in zip(a[0], b[0]) for x, y in zip(bx, by))
    assert all(torch.equal(x, y) for x, y in zip(a[1], b[1]))
    assert not torch.equal(a[1][0], c[1][0]) or not torch.equal(a[0][0].indices, c[0][0].indices)
    u = gs.ops.csr_blocks(*args, fanouts=[25, 10], seed=4, call=7, entry_offsets=True)
    assert not all(torch.equal(x, y) for x, y in zip(a[1], u[1]))


def test_argument_errors(gs):
    indptr, indices = graph("messy")
    with pytest.raises(TypeError, match="sample_weights"):
        gs.ops.csr_blocks(dev(indptr), dev(indices), dev(np.array([1], np.int32)), 1, fanouts=[3],
                          sample_weights=dev(np.ones(len(indices))))
    with pytest.raises(ValueError, match="one weight per CSR entry"):
        gs.ops.csr_blocks(dev(indptr), dev(indices), dev(np.array([1], np.int32)), 1, fanouts=[3],
                          sample_weights=dev(np.ones(len(indices) + 1, np.float32)))
    with pytest.raises(ValueError, match="one weight per CSR entry"):
        gs.ops.sample_csr_rows(dev(indptr), dev(indices), 3, 0, 0, 0, weights=dev(np.ones(3, np.float32)))


# ---------------------------------------------------------------- the law on the GPU
@pytest.mark.parametrize("weights", [[1, 2, 3, 4, 5, 6], [0.5, 8, 1, 0.25, 3, 2]])
def test_inclusion_frequencies_on_the_gpu(gs, weights):
    n, d, k = 1 << 20, 6, 3
    indptr = dev(np.arange(n + 1, dtype=np.int64) * d)
    indices = dev(np.tile(np.arange(d, dtype=np.int32), n))
    w = dev(np.tile(np.asarray(weights, np.float32), n))
    ptr, idx = gs.ops.sample_csr_rows(indptr, indices, k, 31, 2, 0, weights=w)
    assert torch.equal(torch.diff(ptr), torch.full((n,), k, dtype=torch.int64, device="cuda"))
    code = (1 << idx.long().view(n, k)).sum(dim=1)
    counts = torch.bincount(code, minlength=64).cpu().numpy()
    w64 = np.asarray(weights, np.float64)
    probs = {}
    for seq in itertools.permutations(range(d), k):
        left, q = w64.sum(), 1.0
        for j in seq:
            q *= w64[j] / left
            left -= w64[j]
        c = sum(1 << j for j in seq)
        probs[c] = probs.get(c, 0.0) + q
    assert sum(counts[c] for c in probs) == n
    for c, p in probs.items():
        assert abs(counts[c] - n * p) < 5 * np.sqrt(n * p * (1 - p)), (bin(c), counts[c], n * p)


# ---------------------------------------------------------------- the models
IDS = np.array([0, 5, 299, 17, 17, 4, 150, 6, 1, 2, 3, -1], dtype=np.int32)
MODEL_CASES = [("mean", True, "fp32", 0, 2, 5), ("gcn", False, "fp32", 16, 2, 10), ("maxpool", True, "fp32", 0, 2, 3),
               ("meanpool", False, "fp32", 16, 2, 25), ("mean", False, "tf32x3", 16, 3, 4), ("maxpool", False, "fp32",
                                                                                            0, 1, 1)]


def _labels(n):
    return np.eye(4, dtype=np.float32)[np.arange(n) % 4]


def _check(m, rl, loss, grads, head, demb):
    assert abs(float(loss) - rl) < GRAD_TOL * max(1.0, abs(rl))
    for (l, k), v in named_grads(m):
        ref = head[k] if l == "head" else grads[l][k]
        tol = POOL_BIAS_TOL if k == "mlp_bias" else GRAD_TOL
        assert rel_err(v.grad.cpu().numpy(), ref) < tol, (l, k, rel_err(v.grad.cpu().numpy(), ref))
    if demb is not None:
        assert rel_err(m.embeds.grad.cpu().numpy(), demb) < GRAD_TOL


@pytest.mark.parametrize("kind,concat,math,identity_dim,layers,fanout", MODEL_CASES)
@pytest.mark.parametrize("edge", ["none", "same", "other"])
def test_embeddings_losses_and_gradients_match_the_oracle(gs, kind, concat, math, identity_dim, layers, fanout, edge):
    m = sup_model(gs, kind, concat, math, "fp32", identity_dim, layers, fanout=fanout)
    indptr, indices = edge_csr(np.random.RandomState(1), 300, 300)
    sw = weights_of(len(indices), "mixed", 3)
    ew = {"none": None, "same": sw, "other": weights_of(len(indices), "positive", 4)}[edge]
    if edge == "same":                                         # one finite tensor for both: zeros are never drawn
        sw = ew = weights_of(len(indices), "zeros", 3)
    d_sw, d_ew = dev(sw), (None if ew is None else dev(ew))
    sampler = m.layer_infos[0].neigh_sampler
    fanouts = [info.num_samples for info in m.layer_infos]
    feats = m.features.float().cpu().numpy()
    call = int(sampler.counter)
    emb = m.sampled_minibatch_embeddings(dev(indptr), dev(indices), IDS, edge_weight=d_ew, sample_weight=d_sw)
    assert sampler.counter == call + 1
    want = ws.embeddings(feats, indptr, indices, sw, oracle_aggs(m), concat, IDS, fanouts, sampler.seed, call,
                         edge_weight=ew)
    assert rel_err(emb.cpu().numpy(), want) < 1e-4
    call = int(sampler.counter)
    labels = _labels(len(IDS))
    m.optimizer.zero_grad(set_to_none=True)
    loss = m.sampled_minibatch_loss(dev(indptr), dev(indices), IDS, labels, edge_weight=d_ew,
                                    sample_weight=sw if edge == "none" else d_sw)          # numpy is uploaded
    loss.backward()
    rl, grads, head, demb = ws.loss_grads(feats, indptr, indices, sw, oracle_aggs(m), concat, IDS, labels,
                                          m.node_pred_vars["weights"].detach().cpu().numpy(),
                                          m.node_pred_vars["bias"].detach().cpu().numpy(), fanouts, sampler.seed, call,
                                          m.sigmoid_loss, m.weight_decay, identity_dim, edge_weight=ew)
    _check(m, rl, loss.detach(), grads, head, demb)


@pytest.mark.parametrize("kind,concat,math,identity_dim,layers,fanout", MODEL_CASES)
def test_dropout_matches_the_oracle(gs, kind, concat, math, identity_dim, layers, fanout, monkeypatch):
    m = sup_model(gs, kind, concat, math, "fp32", identity_dim, layers, fanout=fanout)
    indptr, indices = edge_csr(np.random.RandomState(1), 300, 300)
    sw = weights_of(len(indices), "heavy", 5)
    sampler = m.layer_infos[0].neigh_sampler
    call = int(sampler.counter)
    m.dropout_counter = 13
    feats = m.features.float().cpu().numpy()
    loss = m.sampled_minibatch_loss(dev(indptr), dev(indices), IDS, _labels(len(IDS)), dropout=0.4,
                                    sample_weight=dev(sw))
    loss.backward()
    fanouts = [info.num_samples for info in m.layer_infos]
    # the dropout oracle over the weighted blocks: its masks name entries by raw CSR position, which the blocks keep
    monkeypatch.setattr(sbd, "_blocks_and_maps", lambda ip, ix, seeds, fan, seed, c:
                        ws.blocks_and_maps(ip, ix, sw, seeds, fan, seed, c))
    rl, grads, head, demb = sbd.sampled_loss_grads_dropout(
        feats, indptr, indices, oracle_aggs(m), concat, IDS, _labels(len(IDS)),
        m.node_pred_vars["weights"].detach().cpu().numpy(), m.node_pred_vars["bias"].detach().cpu().numpy(), fanouts,
        sampler.seed, call, fd.sites(kind, layers, True, m.dropout_key, 13, 0.4), False, m.weight_decay, identity_dim)
    _check(m, rl, loss.detach(), grads, head, demb)


@pytest.mark.parametrize("kind", ["mean", "gcn", "maxpool", "meanpool"])
def test_invariants(gs, kind):
    indptr, indices = capped_csr()
    d_ip, d_ix = dev(indptr), dev(indices)
    sw = dev(weights_of(len(indices), "heavy", 6))
    labels = _labels(len(IDS))
    concat = kind != "gcn"
    # sample_weight=None is the uniform path, bit for bit
    a, b = sup_model(gs, kind, concat, identity_dim=8), sup_model(gs, kind, concat, identity_dim=8)
    la = a.sampled_minibatch_loss(d_ip, d_ix, IDS, labels, sample_weight=None)
    lb = b.sampled_minibatch_loss(d_ip, d_ix, IDS, labels)
    la.backward()
    lb.backward()
    assert torch.equal(la, lb) and all(torch.equal(p.grad, q.grad) for p, q in zip(a.parameters(), b.parameters()))
    # positive weights and fanouts >= every degree: the whole-neighbourhood minibatch
    _set_fanouts(a, 256)
    emb = a.sampled_minibatch_embeddings(d_ip, d_ix, IDS, sample_weight=sw)
    assert torch.equal(emb, a.full_neighbor_minibatch_embeddings(d_ip, d_ix, IDS))
    # with dropout the masks follow the raw positions: the uniform large-fanout blocks are the same blocks
    c = sup_model(gs, kind, concat, identity_dim=8)
    _set_fanouts(c, 256)
    _set_fanouts(b, 256)
    for m in (b, c):
        m.dropout_counter = 3
        m.optimizer.zero_grad(set_to_none=True)
    lc = c.sampled_minibatch_loss(d_ip, d_ix, IDS, labels, dropout=0.3, sample_weight=sw, edge_weight=None)
    lb = b.sampled_minibatch_loss(d_ip, d_ix, IDS, labels, dropout=0.3)
    lc.backward()
    lb.backward()
    assert torch.equal(lc, lb) and all(torch.equal(p.grad, q.grad) for p, q in zip(c.parameters(), b.parameters()))
    # one counter step and one host read per block set, the size read the uniform blocks make too
    sampler = c.layer_infos[0].neigh_sampler
    before = int(sampler.counter)
    _set_fanouts(c, 5)
    ids, d_labels = dev(IDS), dev(labels)
    c.sampled_minibatch_loss(d_ip, d_ix, ids, d_labels, sample_weight=sw).backward()
    assert sampler.counter == before + 1
    torch.cuda.set_sync_debug_mode("warn")
    torch.cuda.set_sync_debug_mode("default")
    reads = []
    for kw in ({}, {"sample_weight": sw}):
        torch.cuda.synchronize()
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter("always")
            torch.cuda.set_sync_debug_mode("warn")
            try:
                c.sampled_minibatch_loss(d_ip, d_ix, ids, d_labels, **kw).backward()
            finally:
                torch.cuda.set_sync_debug_mode("default")
        reads.append([(x.filename.split("/")[-1], x.lineno) for x in w if "synchroniz" in str(x.message)])
    assert len(reads[1]) == 1 and reads[1] == reads[0], reads


@pytest.mark.parametrize("twin", ["host-fp32", "host-bf16", "host-int8", "int8"])
def test_host_and_int8_tables_give_the_device_bits(gs, twin):
    indptr, indices = edge_csr(np.random.RandomState(1), 300, 300)
    sw = dev(weights_of(len(indices), "mixed", 7))
    ew = dev(weights_of(len(indices), "positive", 8))
    m = sup_model(gs, "maxpool", True, "tf32x3", "bf16" if twin == "host-bf16" else "fp32")
    x = m.features.float().cpu()
    if twin == "host-fp32":
        t, ref = gs.HostFeatures(x.numpy(), cache_ids=np.arange(0, 300, 7)), m.features
    elif twin == "host-bf16":
        t, ref = gs.HostFeatures(m.features.cpu(), cache_ids=None), m.features
    elif twin == "host-int8":
        q = gs.Int8Features(x.numpy(), device="cuda")
        t, ref = gs.HostFeatures(gs.Int8Features(x.numpy()), cache_ids=np.arange(0, 300, 3)), q.dequantize()
    else:
        t = gs.Int8Features(x.numpy(), device="cuda")
        ref = t.dequantize()
    sampler = m.layer_infos[0].neigh_sampler
    out = []
    for table in (ref, t):
        m.features = table
        sampler.counter = 4
        m.optimizer.zero_grad(set_to_none=True)
        emb = m.sampled_minibatch_embeddings(dev(indptr), dev(indices), IDS, sample_weight=sw, edge_weight=ew)
        loss = m.sampled_minibatch_loss(dev(indptr), dev(indices), IDS, _labels(len(IDS)), sample_weight=sw,
                                        edge_weight=ew)
        loss.backward()
        out.append((emb, loss.detach(), [p.grad.clone() for p in m.parameters() if p.grad is not None]))
    assert torch.equal(out[0][0], out[1][0]) and torch.equal(out[0][1], out[1][1])
    assert all(torch.equal(a, b) for a, b in zip(out[0][2], out[1][2]))


def test_unsupervised_loss_matches_the_uniform_large_fanout_loss(gs):
    indptr, indices = capped_csr()
    sw = dev(weights_of(len(indices), "positive", 9))
    losses = []
    for weighted in (False, True):
        m = unsup_model(gs, "mean")
        _set_fanouts(m, 256)
        b1, b2 = np.arange(0, 16, dtype=np.int32), np.arange(16, 32, dtype=np.int32)
        kw = {"sample_weight": sw} if weighted else {}
        loss = m.sampled_minibatch_loss(dev(indptr), dev(indices), b1, b2, **kw)
        loss.backward()
        losses.append((loss.detach(), [p.grad.clone() for p in m.parameters() if p.grad is not None]))
        step = m.sampled_minibatch_train_step(dev(indptr), dev(indices), b1, b2, **kw)
        losses[-1] += (step,)
    assert torch.equal(losses[0][0], losses[1][0]) and torch.equal(losses[0][2], losses[1][2])
    assert all(torch.equal(a, b) for a, b in zip(losses[0][1], losses[1][1]))


def test_five_adam_steps_track_the_cpu_run(gs):
    m = sup_model(gs, "mean", identity_dim=8)
    indptr, indices = edge_csr(np.random.RandomState(2), 300, 300)
    sw = weights_of(len(indices), "heavy", 10)
    ids = np.arange(0, 300, 3, dtype=np.int32)
    labels = _labels(len(ids))
    fanouts = [info.num_samples for info in m.layer_infos]
    sampler = m.layer_infos[0].neigh_sampler
    start = int(sampler.counter)
    cpu = [p.detach().cpu().clone().requires_grad_(True) for p in m.parameters()]
    opt = torch.optim.Adam(cpu, lr=m.learning_rate)
    for step in range(5):
        for p, c in zip(m.parameters(), cpu):
            with torch.no_grad():
                p.copy_(c.detach().to(p.device))
        rl, grads, head, demb = ws.loss_grads(m.features.float().cpu().numpy(), dev(indptr).cpu().numpy(), indices,
                                              sw, oracle_aggs(m), m.concat, ids, labels,
                                              m.node_pred_vars["weights"].detach().cpu().numpy(),
                                              m.node_pred_vars["bias"].detach().cpu().numpy(), fanouts, sampler.seed,
                                              start + step, m.sigmoid_loss, m.weight_decay, m.identity_dim)
        refs = {id(v): (head[k] if l == "head" else grads[l][k]) for (l, k), v in named_grads(m)}
        refs[id(m.embeds)] = demb
        for p, c in zip(m.parameters(), cpu):
            c.grad = torch.from_numpy(np.asarray(refs[id(p)], np.float32)).clamp(-5.0, 5.0)
        opt.step()
    m2 = sup_model(gs, "mean", identity_dim=8)
    m2.layer_infos[0].neigh_sampler.counter = start
    for _ in range(5):
        loss = m2.sampled_minibatch_train_step(dev(indptr), dev(indices), ids, labels, sample_weight=dev(sw))
    assert loss.dim() == 0 and loss.is_cuda and m2.layer_infos[0].neigh_sampler.counter == start + 5
    for p, c in zip(m2.parameters(), cpu):
        assert rel_err(p.detach().cpu().numpy(), c.detach().numpy()) < 1e-2


def test_refusals(gs):
    m = sup_model(gs, "mean")
    indptr, indices = edge_csr(np.random.RandomState(1), 300, 300)
    sw = weights_of(len(indices), "positive")
    labels = _labels(len(IDS))
    with pytest.raises(NotImplementedError, match="edge_weight with training dropout"):
        m.sampled_minibatch_loss(indptr, indices, IDS, labels, dropout=0.5, edge_weight=sw, sample_weight=sw)
    with pytest.raises(ValueError, match="device"):
        m.sampled_minibatch_embeddings(indptr, indices, IDS, sample_weight=torch.from_numpy(sw))
    with pytest.raises(ValueError, match="sample_weight needs one weight per CSR entry"):
        m.sampled_minibatch_embeddings(indptr, indices, IDS, sample_weight=sw[:-1])
    with pytest.raises(TypeError, match="sample_weight must be float32"):
        m.sampled_minibatch_embeddings(indptr, indices, IDS, sample_weight=sw.astype(np.float64))
    for name in ("full_neighbor_embeddings", "full_neighbor_minibatch_embeddings"):
        with pytest.raises(TypeError):
            getattr(m, name)(indptr, indices, IDS, sample_weight=sw)
    m.features = gs.Int8Features(m.features.float())
    with pytest.raises(NotImplementedError, match="dropout"):
        m.sampled_minibatch_loss(indptr, indices, IDS, labels, dropout=0.5, sample_weight=sw)
