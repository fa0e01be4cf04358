"""GPU: the LSTM sequence aggregator's kernels (csrc/lstm.cu) through the C ABI, against the teacher-forced float64
references of oracle/seq.py (lstm_step_reference / lstm_bptt_step_reference, whose bounds are derived there and shown to
reject subtly wrong kernels in tests/test_seq_numerics_cpu.py): every saved row of gs_lstm_forward and every dZ row of
gs_lstm_backward, across tile boundaries (S = 32 sequences per CTA at H = 128, 16 at H = 256) up to the bench's hop-2
count of 5,120 sequences and one more, k up to 128, tiles that end before k, clamped and non-positive lengths,
saturated gates and NaN-padded strided operands; gs_seq_lengths past its grid cap; and the seq aggregator at the
Reddit shape (B = 512, fanout 25 x 10, F = 602) against the float64 oracle, one supervised step against float64
autograd."""
import numpy as np
import pytest
import torch

import oracle
from conftest import rel_err
from oracle import seq as oseq

pytestmark = pytest.mark.gpu

TILE = {128: 32, 256: 16}                   # sequences per CTA (SeqTile<H>::kSeqs)
I32_MIN, I32_MAX = -2 ** 31, 2 ** 31 - 1
NAN = float("nan")
# leading-dimension padding per operand for the strided runs (ldw must stay a multiple of 4: the backward's float4 rows)
PADS = dict(P=3, Wh=4, h=1, g=5, c=3, hp=7, dh=2, dZ=1)
NO_PADS = dict.fromkeys(PADS, 0)
PATTERNS = ["ones", "full", "one_long_per_tile", "short_tiles", "above_k", "nonpositive"]


@pytest.fixture(scope="module")
def gs():
    import graphsage_b200
    graphsage_b200._lib.lib()               # raises if the .so is missing: no silent fallback
    return graphsage_b200


def _buf(rows, cols, pad):
    """(full, view): a NaN-filled [rows, cols + pad] buffer and its first `cols` columns.  An output element the kernel
    fails to write stays NaN, and so does a pad column it must not touch."""
    full = torch.full((rows, cols + pad), NAN, dtype=torch.float32, device="cuda")
    return full, full[:, :cols]


def _ld(t):
    return 0 if t is None else t.stride(0)


def _forward(gs, P, Wh, lens, n, k, H, h_last, saved=(None, None, None)):
    L, ptr = gs._lib, gs._lib.ptr
    g, c, hp = saved
    L.check(L.lib().gs_lstm_forward(ptr(P), _ld(P), ptr(Wh), _ld(Wh), ptr(lens), n, k, H, ptr(h_last), _ld(h_last),
                                    ptr(g), _ld(g), ptr(c), _ld(c), ptr(hp), _ld(hp), L.stream_ptr()))


def _backward(gs, dh, g, c, lens, Wh, n, k, H, dZ):
    L, ptr = gs._lib, gs._lib.ptr
    L.check(L.lib().gs_lstm_backward(ptr(dh), _ld(dh), ptr(g), _ld(g), ptr(c), _ld(c), ptr(lens), ptr(Wh), _ld(Wh), n, k, H,
                                     ptr(dZ), _ld(dZ), L.stream_ptr()))


def _n(label, H):
    S = TILE[H]
    return {"1": 1, "S-1": S - 1, "S": S, "S+1": S + 1}.get(label, label)


def _lengths(pattern, n, k, S, rs):
    tile = np.arange(n) // S
    first = np.arange(0, n, S)                                        # the first sequence of each tile
    if pattern == "ones":
        L = np.ones(n)
    elif pattern == "full":
        L = np.full(n, k)
    elif pattern == "one_long_per_tile":                              # one sequence of length k per tile, the rest 1
        L = np.ones(n)
        L[np.minimum(first + rs.randint(0, S, size=len(first)), n - 1)] = k
    elif pattern == "short_tiles":                                    # even tiles end before k: the `t >= tl` branch
        L = rs.randint(1, k + 1, size=n)
        L[first[1::2]] = k
        short = tile % 2 == 0
        L[short] = rs.randint(1, k, size=short.sum()) if k > 1 else 0
    elif pattern == "above_k":                                        # clamped to k
        L = rs.randint(1, k + 1, size=n)
        big = rs.rand(n) < 0.4
        L[big] = rs.choice([k + 1, k + 1000, I32_MAX], size=big.sum())
    elif pattern == "nonpositive":                                    # behave as 0; tile 0 has no sequence that runs
        L = rs.randint(1, k + 1, size=n)
        neg = (rs.rand(n) < 0.25) | (tile == 0)
        L[neg] = rs.choice([0, -1, -k, I32_MIN], size=neg.sum())
    else:
        raise ValueError(pattern)
    return L.astype(np.int32)


def _subset(n, S):
    """The sequences checked on the host: all of them for up to four tiles, else tiles 0, 1, the middle one and the
    last two (the ragged one included).  Every sequence of every tile is still checked on the device for writes,
    exact zeros past len and determinism."""
    T = (n + S - 1) // S
    tiles = range(T) if T <= 4 else sorted({0, 1, T // 2, T - 2, T - 1})
    return np.concatenate([np.arange(t * S, min((t + 1) * S, n)) for t in tiles])


def _host(view, idx, k):
    rows = (torch.from_numpy(idx).cuda()[:, None] * k + torch.arange(k, device="cuda")[None, :]).reshape(-1)
    return view.index_select(0, rows).cpu().numpy().reshape(len(idx), k, -1)


def _run_case(gs, H, n, k, pattern, seed, pad=False, saturate=False):
    """Runs forward (with and without training outputs) and backward twice on NaN-prefilled buffers and checks them;
    returns (worst ratios, host arrays of the checked subset)."""
    S, pads = TILE[H], (PADS if pad else NO_PADS)
    rs = np.random.RandomState(seed)
    lengths = _lengths(pattern, n, k, S, rs)
    lens = torch.from_numpy(lengths).cuda()
    gen = torch.Generator(device="cuda").manual_seed(seed)
    Wf, Wh = _buf(H, 4 * H, pads["Wh"])
    r = np.sqrt(6.0 / (50 + 5 * H))                                   # glorot for K = 50
    Wh.uniform_(-r, r, generator=gen)
    Pf, P = _buf(n * k, 4 * H, pads["P"])
    P.normal_(0.0, 0.8, generator=gen)
    if saturate:                                                      # every third unit of each gate: |z| to 100+
        cols = (torch.arange(4 * H, device="cuda") % H) % 3 == 0
        P[:, cols] = P[:, cols] * 60
    Lc = lens.long().clamp(0, k)
    off = (torch.arange(k, device="cuda")[None, :] >= Lc[:, None]).reshape(-1)
    P[off] = NAN                                                      # never read: the LSTM stops at len
    dhf, dh = _buf(n, H, pads["dh"])
    dh.normal_(0.0, 1.0, generator=gen)
    dh[Lc == 0] = NAN                                                 # a sequence that runs no step reads no dh_last

    def fwd():
        bufs = [_buf(n, H, pads["h"]), _buf(n * k, 4 * H, pads["g"]), _buf(n * k, H, pads["c"]), _buf(n * k, H, pads["hp"])]
        _forward(gs, P, Wh, lens, n, k, H, bufs[0][1], tuple(b[1] for b in bufs[1:]))
        return bufs

    out = fwd()
    (hf, h), (gf, g), (cf, c), (hpf, hp) = out
    hof, h_only = _buf(n, H, pads["h"])
    _forward(gs, P, Wh, lens, n, k, H, h_only)
    zf, dZ = _buf(n * k, 4 * H, pads["dZ"])
    _backward(gs, dh, g, c, lens, Wh, n, k, H, dZ)
    # bit-identical: training outputs or not, and a second call
    assert torch.equal(h_only, h)
    again = fwd()
    assert all(torch.equal(a[1], b[1]) for a, b in zip(out, again))
    del again
    z2f, dZ2 = _buf(n * k, 4 * H, pads["dZ"])
    _backward(gs, dh, g, c, lens, Wh, n, k, H, dZ2)
    assert torch.equal(dZ, dZ2)
    del z2f, dZ2
    # every element written and finite; rows past len exact zeros; pad columns untouched
    for name, v in (("h_last", h), ("gates", g), ("c", c), ("h_prev", hp), ("dZ", dZ)):
        assert bool(torch.isfinite(v).all()), name
    for name, v in (("gates", g), ("c", c), ("h_prev", hp), ("dZ", dZ)):
        assert not bool(v[off].any()), name
    assert not bool(h[Lc == 0].any())
    if pad:
        for name, (f, w) in (("h_last", (hf, H)), ("gates", (gf, 4 * H)), ("c", (cf, H)), ("h_prev", (hpf, H)),
                             ("dZ", (zf, 4 * H)), ("h_only", (hof, H))):
            assert bool(torch.isnan(f[:, w:]).all()), name
    # the teacher-forced bounds on the host
    idx = _subset(n, S)
    host = dict(P=_host(P, idx, k), g=_host(g, idx, k), c=_host(c, idx, k), hp=_host(hp, idx, k), dZ=_host(dZ, idx, k),
                h=h.cpu().numpy()[idx], dh=dh.cpu().numpy()[idx], L=lengths[idx], Wh=Wh.cpu().numpy())
    okf, worst = oseq.check_lstm_forward(host["P"], host["Wh"], host["L"], host["h"], host["g"], host["c"], host["hp"])
    okb, worst["dZ"] = oseq.check_lstm_backward(host["dh"], host["g"], host["c"], host["L"], host["Wh"], host["dZ"])
    print("RATIOS H=%d n=%d k=%d %s%s%s: %s" % (H, n, k, pattern, " pad" if pad else "", " saturate" if saturate else "",
                                                " ".join("%s=%.3f" % kv for kv in worst.items())))
    assert okf and okb, worst
    return worst, host


@pytest.mark.parametrize("pattern", PATTERNS)
@pytest.mark.parametrize("k", [1, 2, 25, 128])
@pytest.mark.parametrize("n", ["1", "S-1", "S", "S+1"])
@pytest.mark.parametrize("H", [128, 256])
def test_lstm_kernels_against_teacher_forced_bounds(gs, H, n, k, pattern):
    _run_case(gs, H, _n(n, H), k, pattern, seed=1000 * k + 10 * PATTERNS.index(pattern) + _n(n, H))


@pytest.mark.parametrize("pattern", ["short_tiles", "nonpositive"])
@pytest.mark.parametrize("k", [25, 128])
@pytest.mark.parametrize("n", [5120, 5121])
@pytest.mark.parametrize("H", [128, 256])
def test_lstm_kernels_many_tiles(gs, H, n, k, pattern):
    """160 / 320 CTAs at n = 5,120 (the bench's hop-2 count) and a ragged last tile of one sequence at 5,121."""
    _run_case(gs, H, n, k, pattern, seed=n + k)


@pytest.mark.parametrize("n,k", [("S+1", 25), (5121, 2)])
@pytest.mark.parametrize("H", [128, 256])
def test_lstm_kernels_strided_nan_padded_operands(gs, H, n, k):
    """Every operand in a buffer wider than its row (ldp, ldw, ldh, ldg, ldc, ldhp, lddh, ldz all above the minimum),
    the pad columns NaN: a pad column read shows up as NaN in the results, one written loses its NaN."""
    _run_case(gs, H, _n(n, H), k, "above_k", seed=7 + k, pad=True)


@pytest.mark.parametrize("k", [25, 128])
@pytest.mark.parametrize("H", [128, 256])
def test_lstm_kernels_saturated_gates(gs, H, k):
    """|z| of 30 - 100+ on every third unit: sigmoid reaches exactly 0 and 1 in fp32, tanh exactly +-1, and the
    backward's sigma (1 - sigma) and 1 - tanh^2 factors exactly 0."""
    worst, host = _run_case(gs, H, TILE[H] + 1, k, "short_tiles", seed=3 + k, saturate=True)
    n = len(host["L"])
    on = (np.arange(k)[None, :] < np.clip(host["L"], 0, k)[:, None])[:, :, None]
    c_prev = np.concatenate([np.zeros((n, 1, H)), host["c"][:, :-1]], axis=1)
    ref = oseq.lstm_step_reference(host["P"], host["Wh"], host["hp"], c_prev, host["L"])["gates"][0]
    tanh_col = np.arange(4 * H) // H == 1
    deep1 = on & (np.abs(ref) == 1.0)                                 # saturated beyond float64's resolution
    deep0 = on & ~tanh_col & (ref <= 2.0 ** -140)                     # expf(-z) overflows: sigmoid is exactly 0
    assert deep1.sum() > 100 and deep0.sum() > 10
    assert np.array_equal(host["g"][deep1], np.sign(ref[deep1]))
    assert not host["g"][deep0].any()
    sat = oseq.saturated(host["g"]) & on
    assert not host["dZ"][sat].any()


@pytest.mark.parametrize("K", [1, 33, 602])
def test_seq_lengths_past_the_grid_cap(gs, K):
    """n = 20,000 sequences, above the kernel's grid (8 warps x 8 CTAs per SM), so warps loop; rows of ldx = 608 whose
    pad columns past K are non-zero and must not count; -0.0 rows, rows whose only non-zero element is a subnormal
    (+-1e-45: the library is built without flush-to-zero), zero rows and all-zero sequences (length 1)."""
    n, k, ld = 20000, 5, 608
    assert n > torch.cuda.get_device_properties(0).multi_processor_count * 64
    rs = np.random.RandomState(K)
    x = rs.randn(n * k, ld).astype(np.float32)
    x[:, K:] = 1.0
    kind = rs.randint(0, 5, size=n * k)
    kind[:10 * k] = 3                                                 # sequences 0 - 9: nothing but zero rows
    x[kind == 1, :K] = -0.0
    sub = np.flatnonzero(kind == 2)
    x[sub, :K] = 0.0
    x[sub, rs.randint(0, K, size=len(sub))] = rs.choice(np.array([1e-45, -1e-45], np.float32), size=len(sub))
    x[kind == 3, :K] = 0.0
    xd = torch.from_numpy(x).cuda()
    got = gs.ops.seq_lengths(xd[:, :K], n, k).cpu().numpy()
    want = oseq.seq_lengths(x[:, :K].reshape(n, k, K))
    assert np.array_equal(got, want)
    assert np.all(got[:10] == 1) and got.max() == k and len(np.unique(got)) == k


# ---------------------------------------------------------------- the aggregator at the Reddit shape
@pytest.fixture(scope="module")
def reddit(gs):
    from graphsage_b200.synthetic import reddit_like
    g = reddit_like(n=232965, f=602, max_degree=128, seed=123)
    P = gs.ops.pad_cols(602)
    table = torch.zeros((g["n"] + 1, P), dtype=torch.float32, device="cuda")
    table[:, :602] = torch.from_numpy(g["features"]).cuda()
    g["table"] = table
    g["adj_dev"] = torch.from_numpy(g["adj"]).cuda()
    return g


def _oracle_aggs(aggs, dtype=np.float64):
    return [dict(kernel=a.cell.vars["kernel"].detach().cpu().numpy().astype(dtype),
                 cell_bias=a.cell.vars["bias"].detach().cpu().numpy().astype(dtype),
                 neigh_weights=a.vars["neigh_weights"].detach().cpu().numpy().astype(dtype),
                 self_weights=a.vars["self_weights"].detach().cpu().numpy().astype(dtype)) for a in aggs]


def _perturb_cell_bias(m, seed):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    for a in m.aggregators:                                           # zero biases leave the gates symmetric
        a.cell.vars["bias"].data.add_(torch.randn(a.cell.vars["bias"].shape, generator=gen, device="cuda") * 0.2)


@pytest.mark.parametrize("math", ["fp32", "tf32x3"])
@pytest.mark.parametrize("size,concat", [("small", True), ("big", False)])
def test_reddit_shaped_forward_vs_oracle(gs, reddit, size, concat, math):
    """B = 512, fanout 25 x 10, F = 602: 5,120 hop-1 and 128,000 hop-2 rows, H = 128 (small) / 256 (big).  The float64
    oracle takes seconds of CPU time here, so "big" runs at the full B as well."""
    g, B = reddit, 512
    gs.inits.manual_seed(21)
    gs.set_default_math(math)
    try:
        sampler = gs.UniformNeighborSampler(g["adj_dev"], seed=123)
        infos = [gs.SAGEInfo("node", sampler, 25, 128), gs.SAGEInfo("node", sampler, 10, 128)]
        m = gs.SampleAndAggregate({"batch_size": B, "dropout": 0.}, g["table"][:, :602], g["adj_dev"], None, infos,
                                  concat=concat, aggregator_type="seq", model_size=size)
        seeds = np.random.RandomState(1).randint(0, g["n"], size=B).astype(np.int32)
        m.forward(torch.from_numpy(seeds), normalize=False)          # creates the aggregators
        _perturb_cell_bias(m, 5)
        c0 = sampler.counter
        out = m.forward(torch.from_numpy(seeds), normalize=False).cpu().numpy()
    finally:
        gs.set_default_math("fp32")
    samples, support = oracle.sample_khop(g["adj"], seeds, [25, 10], 123, c0)
    ref = oseq.aggregate_khop_seq(samples, g["features"], [25, 10], support, B, _oracle_aggs(m.aggregators), concat,
                                  dtype=np.float64)
    err = rel_err(out, ref)
    print("seq Reddit-shaped forward %s %s: rel_err %.2e" % (size, math, err))
    assert err < 1e-4, err


def test_reddit_shaped_supervised_step_vs_float64_autograd(gs, reddit):
    """One supervised step at B = 64, fanout 25 x 10, F = 602: the loss and every gradient (the cell's kernel and bias
    through gs_lstm_backward) against torch float64 autograd on oracle.seq.torch_seq_layer."""
    g, B, Cn, wd = reddit, 64, 41, 1e-3
    gs.inits.manual_seed(22)
    sampler = gs.UniformNeighborSampler(g["adj_dev"], seed=123)
    infos = [gs.SAGEInfo("node", sampler, 25, 128), gs.SAGEInfo("node", sampler, 10, 128)]
    m = gs.SupervisedGraphsage(Cn, {"batch_size": B, "dropout": 0.}, g["table"][:, :602], g["adj_dev"], None, infos,
                               concat=True, aggregator_type="seq", sigmoid_loss=True, learning_rate=0.01, weight_decay=wd)
    _perturb_cell_bias(m, 6)
    aggs = [{key: v.detach().cpu().double().clone().requires_grad_(True) for key, v in
             dict(kernel=a.cell.vars["kernel"], cell_bias=a.cell.vars["bias"], **a.vars).items()} for a in m.aggregators]
    head = {key: v.detach().cpu().double().clone().requires_grad_(True) for key, v in m.node_pred_vars.items()}
    cpu_params = [a[key] for a in aggs for key in ("neigh_weights", "self_weights")] + \
        [a[key] for a in aggs for key in ("kernel", "cell_bias")] + list(head.values())
    rs = np.random.RandomState(6)
    seeds = rs.randint(0, g["n"], size=B).astype(np.int32)
    labels = (rs.rand(B, Cn) < 0.3).astype(np.float32)
    c0 = sampler.counter
    m.optimizer.zero_grad(set_to_none=True)
    loss = m.loss(torch.from_numpy(seeds), torch.from_numpy(labels))
    loss.backward()
    loss = loss.detach()
    samples, _ = oracle.sample_khop(g["adj"], seeds, [25, 10], 123, c0)
    hidden = [torch.from_numpy(g["features"][np.asarray(s)].astype(np.float64)) for s in samples]
    fan = [25, 10]
    for layer in range(2):
        a = aggs[layer]
        hidden = [oseq.torch_seq_layer(hidden[hop], hidden[hop + 1], a["kernel"], a["cell_bias"], a["self_weights"],
                                       a["neigh_weights"], fan[1 - hop], True, layer == 1) for hop in range(2 - layer)]
    out = hidden[0]
    out = out / torch.sqrt(torch.clamp((out * out).sum(dim=1, keepdim=True), min=1e-12))
    ref = torch.nn.functional.binary_cross_entropy_with_logits(out @ head["weights"] + head["bias"],
                                                               torch.from_numpy(labels).double())
    for t in [a["neigh_weights"] for a in aggs] + [a["self_weights"] for a in aggs] + list(head.values()):
        ref = ref + wd * 0.5 * (t * t).sum()                          # the cell's kernel and bias are not decayed
    ref.backward()
    ref = ref.detach()
    assert abs(float(loss) - float(ref)) < 2e-4 * max(1.0, abs(float(ref)))
    errs = [rel_err(p.grad.cpu().numpy().reshape(1, -1), q.grad.numpy().reshape(1, -1), floor=1e-8)
            for p, q in zip(m.parameters(), cpu_params)]
    print("seq Reddit-shaped supervised step: loss %.6f vs %.6f, gradient rel_err max %.2e"
          % (float(loss), float(ref), max(errs)))
    assert len(errs) == len(cpu_params) and max(errs) < 2e-4, errs
