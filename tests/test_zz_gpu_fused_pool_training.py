"""GPU: training the max-pool / mean-pool branch through the fused bf16 kernels (fused_pool=True).

B1 (gs_pool_mlp_backward_dp) is checked bit for bit against oracle/pool_grad.py on grid-valued inputs (multiples of 2^-4:
exact in bf16, and every fp32 sum of their products is exact), B2 / B3 against fp64 products of the kernel's own dP
within oracle/numerics.py's GEMM bounds, and the whole step against torch-CPU autograd on bf16-rounded operands with dP
rounded to bf16 where the kernel rounds it.  Also: determinism, CUDA-graph capture, training quality, peak memory and the refusals."""
import numpy as np
import pytest
import torch

from conftest import load_golden
from oracle import numerics as nu
from oracle import pool_grad

pytestmark = pytest.mark.gpu


def _grid(r, shape, lim):
    return (r.randint(-int(lim * 16), int(lim * 16) + 1, size=shape) / 16.0).astype(np.float32)


def _norm_rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))


def _b1_case(pool, k, K, hidden, n, by_ids, seed=0):
    import graphsage_b200 as gs
    r = np.random.RandomState(seed)
    N = 64                                             # few distinct rows: duplicate ids give exact ties
    table = torch.zeros((N + n * k, gs.ops.pad_cols(K)), dtype=torch.bfloat16, device="cuda")
    X_all = _grid(r, (N + n * k, K), 2.0)
    table[:, :K] = torch.from_numpy(X_all).cuda().bfloat16()
    if by_ids:
        ids = r.randint(0, N, size=n * k).astype(np.int32)
        ids[:k] = 5                                    # one group of identical rows
        row_ids, row0, X = torch.from_numpy(ids).cuda(), 0, X_all[ids]
    else:
        row_ids, row0, X = None, 7, X_all[7:7 + n * k]
    W, b = _grid(r, (K, hidden), 1.0), _grid(r, (hidden,), 2.0)
    b[3] = -4096.0                                     # all-negative columns: hp = 0
    b[hidden - 1] = -4096.0
    dhp = _grid(r, (n, hidden), 4.0)
    Wt, bt, dhpt = (torch.from_numpy(v).cuda() for v in (W, b, dhp))
    grad = gs.ops.pool_mlp_backward_dp(table[:, :K], n, k, Wt, bt, gs.ops.PackedMlpWeights(), dhpt, row_ids=row_ids,
                                       row0=row0, K=K, pool=pool)
    pre = (X.astype(np.float64) @ W.astype(np.float64)).astype(np.float32)
    ref = pool_grad.dpre(pre, b, dhp, k, pool)
    return dict(table=table[:, :K], row_ids=row_ids, row0=row0, X=X, W=W, Wt=Wt, grad=grad, ref=ref, n=n, k=k, K=K,
                hidden=hidden)


B1_CASES = [("max", 1, 8, 128, 300, True), ("max", 3, 50, 512, 101, False), ("max", 25, 602, 512, 41, True),
            ("max", 128, 640, 128, 5, True), ("max", 10, 640, 1024, 50, False), ("mean", 3, 602, 1024, 77, True),
            ("mean", 25, 50, 128, 43, False), ("mean", 128, 8, 512, 3, True), ("mean", 1, 640, 512, 129, True),
            ("max", 25, 602, 1024, 1, False)]


@pytest.mark.parametrize("pool,k,K,hidden,n,by_ids", B1_CASES)
def test_b1_matches_the_oracle_bit_for_bit(pool, k, K, hidden, n, by_ids):
    c = _b1_case(pool, k, K, hidden, n, by_ids)
    dP, full, parts = pool_grad.dp_images_to_rows(c["grad"].cpu().numpy(), n, k, hidden)
    assert np.array_equal(dP, pool_grad.bf16_round(c["ref"]))
    assert not full[pool_grad.tile_rows(n, k) < 0].any()          # padding slots are zero
    assert np.array_equal(parts, pool_grad.dbm_partials(c["ref"], n, k))
    if pool == "max":
        assert (c["ref"][:, 3] == 0).all() and (np.abs(c["ref"]) > 0).any()


@pytest.mark.parametrize("pool,k,K,hidden,n,by_ids", [B1_CASES[i] for i in (0, 2, 4, 5, 6, 8)])
def test_b2_b3_match_fp64_products_of_the_kernels_dp(pool, k, K, hidden, n, by_ids):
    import graphsage_b200 as gs
    c = _b1_case(pool, k, K, hidden, n, by_ids, seed=1)
    dP, _, parts = pool_grad.dp_images_to_rows(c["grad"].cpu().numpy(), n, k, hidden)
    dWm = torch.ones((K, hidden), dtype=torch.float32, device="cuda")          # B2 adds into the caller's buffers
    dbm = torch.full((hidden,), 0.5, dtype=torch.float32, device="cuda")
    gs.ops.pool_mlp_backward_dw(c["table"], n, k, c["grad"], dWm, dbm, row_ids=c["row_ids"], row0=c["row0"], K=K)
    dW0 = torch.zeros((K, hidden), dtype=torch.float32, device="cuda")
    gs.ops.pool_mlp_backward_dw(c["table"], n, k, c["grad"], dW0, torch.zeros_like(dbm), row_ids=c["row_ids"],
                                row0=c["row0"], K=K)
    # the sum over the rows is added to dWm once: fl32(1 + the sum), and the sum is held to numerics.check_gemm
    assert np.array_equal(dWm.cpu().numpy(), dW0.cpu().numpy() + np.float32(1))
    _check_dw(dW0, c["X"], dP)
    assert np.array_equal(dbm.cpu().numpy(), (pool_grad.dbm_combine(parts) + np.float32(0.5)).astype(np.float32))
    for d in sorted({K, max(1, K // 3)}):
        dx = gs.ops.pool_mlp_backward_dx(c["grad"], n, k, c["Wt"], gs.ops.PackedMlpDxWeights(d))
        assert tuple(dx.shape) == (n * k, d)
        ok, worst, rms = nu.check_gemm(dx.cpu().numpy(), *nu.gemm_reference([(dP, c["W"].T[:, :d])], "bf16"))
        assert ok, ("B3", d, worst, rms)


def _check_dw(dWm, X, dP):
    """B2's dWm = X^T dP against the fp64 product of its bf16 operands, criteria (a) and (b) of oracle/numerics.py with
    n * k products per element."""
    ok, worst, rms = nu.check_gemm(dWm.cpu().numpy(), *nu.gemm_reference([(X.T, dP)], "bf16"))
    assert ok, ("B2", worst, rms)


@pytest.mark.parametrize("pool,k,K,hidden,n,by_ids", [("max", 1, 50, 128, 5888, True), ("mean", 25, 50, 128, 5000, False),
                                                     ("max", 10, 130, 256, 1010, True)])
def test_b2_many_tiles_uneven_last_chunk_and_dbm_groups(pool, k, K, hidden, n, by_ids):
    """row counts that are not a multiple of B2's chunk: the short last chunk, several dbm groups of 32 tiles"""
    import graphsage_b200 as gs
    blocks, per, chunks = pool_grad.dw_chunks(n, k)
    assert blocks % per != 0 and chunks > 1
    n_tiles = blocks // 2
    assert n_tiles > pool_grad.DBM_GROUP
    c = _b1_case(pool, k, K, hidden, n, by_ids, seed=2)
    dP, _, parts = pool_grad.dp_images_to_rows(c["grad"].cpu().numpy(), n, k, hidden)
    assert np.array_equal(dP, pool_grad.bf16_round(c["ref"]))
    assert np.array_equal(parts, pool_grad.dbm_partials(c["ref"], n, k))
    dWm = torch.zeros((K, hidden), dtype=torch.float32, device="cuda")
    dbm = torch.zeros((hidden,), dtype=torch.float32, device="cuda")
    gs.ops.pool_mlp_backward_dw(c["table"], n, k, c["grad"], dWm, dbm, row_ids=c["row_ids"], row0=c["row0"], K=K)
    _check_dw(dWm, c["X"], dP)
    assert np.array_equal(dbm.cpu().numpy(), pool_grad.dbm_combine(parts))
    # the rows of the last chunk alone: zero dP everywhere else, so a wrong last-chunk bound loses (or doubles) them
    last = np.zeros_like(dP)
    r0 = (chunks - 1) * per * 64                          # first row slot of the last chunk
    keep = pool_grad.tile_rows(n, k).reshape(-1)[r0:]
    keep = keep[keep >= 0]
    last[keep] = dP[keep]
    buf = torch.from_numpy(pool_grad.rows_to_dp_images(last, n, k)).cuda()
    dWm.zero_()
    dbm.zero_()
    gs.ops.pool_mlp_backward_dw(c["table"], n, k, buf, dWm, dbm, row_ids=c["row_ids"], row0=c["row0"], K=K)
    assert np.abs(last).sum() > 0
    _check_dw(dWm, c["X"], last)


def _one_hot_dp(rows, hidden):
    """dP[r, perm(r)] = 1: every row selects one hidden unit, so an output element names the operand element it read"""
    perm = (37 * np.arange(rows) + 5) % hidden
    dP = np.zeros((rows, hidden), np.float32)
    dP[np.arange(rows), perm] = 1.0
    return dP, perm


@pytest.mark.parametrize("hidden", [128, 256])
def test_transposed_a_operand_layout_on_a_known_matrix(hidden):
    """The MN-major (transpose-A) wgmma operand of B2 and B3 on one tile of one-hot rows: every output element is one
    operand element, exactly, so a wrong descriptor or swizzle shows as the exact rows / columns it misplaced."""
    import graphsage_b200 as gs
    r = np.random.RandomState(7)
    n, k, K = 128, 1, 128
    dP, perm = _one_hot_dp(n, hidden)
    buf = torch.from_numpy(pool_grad.rows_to_dp_images(dP, n, k)).cuda()
    W = _grid(r, (K, hidden), 4.0)
    # B3: A = dP^T images read transposed -> dX[r, f] = W[f, perm(r)]
    dx = gs.ops.pool_mlp_backward_dx(buf, n, k, torch.from_numpy(W).cuda(), gs.ops.PackedMlpDxWeights(K)).cpu().numpy()
    want = W[:, perm].T
    bad = np.argwhere(dx != want)
    assert bad.size == 0, ("B3 rows, columns misplaced", bad[:8].tolist())
    # B2: A = X^T (the gathered rows, K4's row image) read transposed -> dWm[f, perm(r)] = X[r, f]
    X = _grid(r, (n, K), 4.0)
    table = torch.zeros((n, K), dtype=torch.bfloat16, device="cuda")
    table[:] = torch.from_numpy(X).cuda().bfloat16()
    dWm = torch.zeros((K, hidden), dtype=torch.float32, device="cuda")
    dbm = torch.zeros((hidden,), dtype=torch.float32, device="cuda")
    gs.ops.pool_mlp_backward_dw(table, n, k, buf, dWm, dbm, row0=0, K=K)
    want = np.zeros((K, hidden), np.float32)
    want[:, perm] = X.T
    bad = np.argwhere(dWm.cpu().numpy() != want)
    assert bad.size == 0, ("B2 (feature, hidden) misplaced", bad[:8].tolist())


def test_dx_pack_refuses_more_columns_than_wm_has():
    import graphsage_b200 as gs
    W = torch.zeros((50, 128), device="cuda")
    with pytest.raises(ValueError, match="cols"):
        gs.ops.PackedMlpDxWeights(51).get(W)


# ---------------------------------------------------------------- whole steps

B, C = 24, 5


def _graph(grid=True):
    g = load_golden("khop")
    feats = torch.from_numpy(g["feats"])
    if grid:
        feats = torch.clamp(torch.round(feats * 16) / 16, -8, 8)
    return torch.from_numpy(g["adj"]).cuda(), feats.cuda()


def _supervised(kind, concat, d, fused=True, cls=None, features=None, sampler_seed=7):
    import graphsage_b200 as gs
    adj, feats = _graph()
    if features is not None:
        feats = features
    gs.inits.manual_seed(11)
    sampler = gs.UniformNeighborSampler(adj, seed=sampler_seed)
    infos = [gs.SAGEInfo("node", sampler, 5, 16), gs.SAGEInfo("node", sampler, 3, 16)]
    if cls is None:
        m = gs.SupervisedGraphsage(C, {"batch_size": B, "dropout": 0.}, feats, adj, None, infos, concat=concat,
                                   aggregator_type=kind, learning_rate=0.01, identity_dim=d, fused_pool=fused)
    else:
        deg = np.ones(adj.shape[0] - 1)
        m = cls({"batch_size": B, "dropout": 0.}, feats, adj, deg, infos, concat=concat, aggregator_type=kind,
                identity_dim=d, neg_sample_size=7, fused_pool=fused)
    gen = torch.Generator(device="cuda").manual_seed(2)
    for a in m.aggregators:
        bias = a.mlp_layers[0].vars["bias"]
        bias.data.add_(torch.randn(bias.shape, generator=gen, device=bias.device) * 0.1)
    return m


def _batch(seed=5, b=B):
    rs = np.random.RandomState(seed)
    ids = torch.from_numpy(rs.randint(0, 300, size=b).astype(np.int32))
    labels = torch.from_numpy(np.eye(C, dtype=np.float32)[rs.randint(0, C, size=b)])
    return ids, labels


class _RoundGrad(torch.autograd.Function):
    """identity forward; the backward rounds the gradient to bf16 (the kernel's dP)"""

    @staticmethod
    def forward(ctx, x):
        return x.clone()

    @staticmethod
    def backward(ctx, g):
        return g.float().bfloat16().double()


def _bf16v(x):
    return x + (x.detach().float().bfloat16().double() - x.detach())


def _ref_outputs(m, P, feats, samples):
    """differentiable_outputs restated in fp64 torch on the CPU, P: the model's parameters as fp64 leaves"""
    L = len(m.layer_infos)
    num = [info.num_samples for info in m.layer_infos]
    hidden = [feats[s.long()] for s in samples]
    for layer in range(L):
        agg = m.aggregators[layer]
        Ws, Wn, Wm, bm = (P[id(v)] for v in (agg.vars["self_weights"], agg.vars["neigh_weights"],
                                             agg.mlp_layers[0].vars["weights"], agg.mlp_layers[0].vars["bias"]))
        nxt = []
        for hop in range(L - layer):
            k = num[L - hop - 1]
            selfv, neigh = hidden[hop], hidden[hop + 1]
            n = selfv.shape[0]
            h = torch.relu(_RoundGrad.apply(_bf16v(neigh) @ _bf16v(Wm)) + bm).reshape(n, k, -1)
            hp = h.amax(dim=1) if agg.pool == "max" else h.mean(dim=1)
            fs, fn = selfv @ Ws, hp @ Wn
            y = torch.cat([fs, fn], dim=1) if agg.concat else fs + fn
            nxt.append(y if layer == L - 1 else torch.relu(y))
        hidden = nxt
    out = hidden[0]
    return out / torch.sqrt(torch.clamp((out * out).sum(dim=1, keepdim=True), min=1e-12))


def _ref_params(m):
    params = m.parameters()
    P = {id(p): p.detach().cpu().double().requires_grad_(True) for p in params}
    return params, P


def _check_grads(params, P, m, feats_leaf, tol=1e-3):
    for p in params:
        if p is getattr(m, "embeds", None):
            ref = feats_leaf.grad[:, :p.shape[1]]
        else:
            ref = P[id(p)].grad
        assert p.grad is not None and ref is not None
        err = _norm_rel(p.grad.cpu().numpy(), ref.numpy())
        assert err <= tol, (tuple(p.shape), err)


@pytest.mark.parametrize("d", [0, 16])
@pytest.mark.parametrize("concat", [True, False])
@pytest.mark.parametrize("kind", ["maxpool", "meanpool"])
def test_supervised_step_matches_cpu_autograd(kind, concat, d):
    _check_supervised_step(_supervised(kind, concat, d))


@pytest.mark.parametrize("kind", ["maxpool", "meanpool"])
def test_supervised_step_over_a_bf16_table_matches_cpu_autograd(kind):
    """a bf16 feature table is K4's operand as it is, and the self rows are widened from it"""
    _, feats = _graph()
    m = _supervised(kind, True, 0, features=feats.bfloat16())
    assert m.features.dtype == torch.bfloat16
    _check_supervised_step(m)


def _check_supervised_step(m):
    from graphsage_b200 import supervised_models as sm
    ids, labels = _batch()
    sampler = m.layer_infos[0].neigh_sampler
    c0 = sampler.counter
    samples, _ = m.sample(ids.cuda(), m.layer_infos, batch_size=B)
    samples = [s.cpu() for s in samples]
    sampler.counter = c0
    params, P = _ref_params(m)
    feats_leaf = m.features.detach().cpu().double().requires_grad_(True)
    loss = m.loss(ids, labels)
    loss.backward()
    out = _ref_outputs(m, P, feats_leaf, samples)
    W, b = P[id(m.node_pred_vars["weights"])], P[id(m.node_pred_vars["bias"])]
    ref = sm.classification_loss(out @ W + b, labels.double(), False)
    ref.backward()
    assert abs(float(loss.detach()) - float(ref.detach())) <= 1e-5 * abs(float(ref.detach()))
    _check_grads(params, P, m, feats_leaf)


def test_unsupervised_step_matches_cpu_autograd():
    import graphsage_b200 as gs
    m = _supervised("maxpool", True, 0, cls=gs.UnsupervisedGraphsage)
    b1, _ = _batch(5)
    b2, _ = _batch(6)
    sampler = m.layer_infos[0].neigh_sampler
    c0, n0 = sampler.counter, m.neg_sampler.counter
    neg = m.neg_sampler(m.neg_sample_size)
    sam = [[s.cpu() for s in m.sample(x.cuda(), m.layer_infos, batch_size=x.numel())[0]] for x in (b1, b2, neg)]
    sampler.counter, m.neg_sampler.counter = c0, n0
    params, P = _ref_params(m)
    feats_leaf = m.features.detach().cpu().double().requires_grad_(True)
    loss = m.loss(b1, b2)
    loss.backward()
    o1, o2, on = (_ref_outputs(m, P, feats_leaf, s) for s in sam)
    ref = m.link_pred_layer.loss(o1, o2, on) / float(o1.shape[0])
    ref.backward()
    assert abs(float(loss.detach()) - float(ref.detach())) <= 1e-5 * abs(float(ref.detach()))
    _check_grads(params, P, m, feats_leaf)


def test_five_steps_twice_are_bit_identical():
    runs = []
    for _ in range(2):
        m = _supervised("maxpool", True, 16)
        for i in range(5):
            m.train_step(*_batch(i))
        runs.append([p.detach().clone() for p in m.parameters()])
    assert all(torch.equal(a, b) for a, b in zip(*runs))


@pytest.mark.parametrize("kind", ["maxpool", "meanpool"])
def test_graphed_step_replays_equal_eager_steps(kind):
    import graphsage_b200 as gs
    m, twin = _supervised(kind, True, 16), _supervised(kind, True, 16)
    gs.make_adam_capturable(twin.optimizer)
    step = m.graphed_train_step(B)
    sizes = [B, B, 11, B]
    for i, b in enumerate(sizes):
        ids, labels = _batch(10 + i, b)
        got = step(ids, labels) if b == B else m.train_step(ids, labels)
        want = twin.train_step(ids, labels)
        assert torch.equal(got, want)
        assert all(torch.equal(p, q) for p, q in zip(m.parameters(), twin.parameters()))
        assert m.layer_infos[0].neigh_sampler.counter == twin.layer_infos[0].neigh_sampler.counter


def test_training_quality_on_toy_ppi_matches_the_materialised_path():
    import graphsage_b200 as gs
    g = load_golden("toy_ppi")
    n = g["feats"].shape[0]
    src = np.concatenate([g["src"], g["dst"]]).astype(np.int64)
    dst = np.concatenate([g["dst"], g["src"]]).astype(np.int64)
    order = np.argsort(src, kind="stable")
    indptr = np.zeros(n + 1, np.int64)
    np.cumsum(np.bincount(src, minlength=n), out=indptr[1:])
    adj, _ = gs.ops.build_padded_adj(torch.from_numpy(indptr).cuda(), torch.from_numpy(dst[order].astype(np.int32)).cuda(), 32)
    feats = torch.zeros((n + 1, 50), dtype=torch.float32, device="cuda")
    feats[:n] = torch.from_numpy(np.asarray(g["feats"], np.float32)).cuda()
    labels_all = (np.asarray(g["labels"]) > 0).astype(np.float32)
    finals = []
    for fused in (False, True):
        gs.inits.manual_seed(3)
        sampler = gs.UniformNeighborSampler(adj, seed=1)
        infos = [gs.SAGEInfo("node", sampler, 10, 64), gs.SAGEInfo("node", sampler, 5, 64)]
        m = gs.SupervisedGraphsage(labels_all.shape[1], {"batch_size": 64, "dropout": 0.}, feats, adj, None, infos,
                                   aggregator_type="maxpool", sigmoid_loss=True, learning_rate=0.01, fused_pool=fused)
        rs = np.random.RandomState(0)
        losses = []
        for _ in range(50):
            ids = rs.randint(0, n, size=64).astype(np.int32)
            losses.append(float(m.train_step(torch.from_numpy(ids), torch.from_numpy(labels_all[ids]))))
        finals.append((losses[0], np.mean(losses[-5:])))
    (l0, lf), (f0, ff) = finals
    assert abs(l0 - f0) <= 1e-2 * l0, finals
    assert lf < l0 and ff < f0
    assert abs(ff - lf) <= 0.05 * abs(lf), finals


def test_peak_memory_is_below_the_materialised_path():
    import graphsage_b200 as gs
    adj, _ = _graph()
    peaks = []
    fan, b, F = (25, 10), 512, 200
    feats = torch.from_numpy(_grid(np.random.RandomState(0), (adj.shape[0], F), 1.0)).cuda()
    for fused in (False, True):
        gs.inits.manual_seed(1)
        sampler = gs.UniformNeighborSampler(adj, seed=1)
        infos = [gs.SAGEInfo("node", sampler, fan[0], 128), gs.SAGEInfo("node", sampler, fan[1], 128)]
        m = gs.SupervisedGraphsage(C, {"batch_size": b, "dropout": 0.}, feats, adj, None, infos, aggregator_type="maxpool",
                                   fused_pool=fused)
        ids, labels = _batch(1, b)
        m.train_step(ids, labels)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        m.train_step(ids, labels)
        torch.cuda.synchronize()
        peaks.append(torch.cuda.max_memory_allocated() - base)
    h_bytes = b * fan[1] * fan[0] * 512 * 4                   # the fp32 h of layer 0's largest hop
    assert peaks[1] + h_bytes <= peaks[0], peaks


def test_refusals_on_the_gpu():
    import graphsage_b200 as gs
    adj, feats = _graph()
    sampler = gs.UniformNeighborSampler(adj, seed=1)
    with pytest.raises(NotImplementedError, match="fanouts <= 128"):
        gs.SupervisedGraphsage(C, {"batch_size": B, "dropout": 0.}, feats, adj, None,
                               [gs.SAGEInfo("node", sampler, 129, 16), gs.SAGEInfo("node", sampler, 3, 16)],
                               aggregator_type="maxpool", fused_pool=True)
    with pytest.raises(NotImplementedError, match="dropout"):
        _supervised_dropout = gs.SupervisedGraphsage(
            C, {"batch_size": B, "dropout": 0.5}, feats, adj, None,
            [gs.SAGEInfo("node", sampler, 5, 16), gs.SAGEInfo("node", sampler, 3, 16)], aggregator_type="meanpool",
            fused_pool=True)
    m = _supervised("maxpool", True, 0)
    with pytest.raises(NotImplementedError, match="dropout"):
        m.loss(*_batch(), dropout=0.3)
