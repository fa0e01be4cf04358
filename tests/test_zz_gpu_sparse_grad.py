"""GPU: the sparse-gradient kernels against the operand-exact contract of oracle/sparse_grad.py.

* gs_embedding_grad and gs_embedding_grad_dropout bit for bit, at d from 1 to 602 (the 128-column tiles of the chunk
  pass past the first included), eight lists with groups 1 / 10 / 25, scales 1, 1/10, 1/26 and -2, an empty list
  between two masked ones, ids -1, n_rows and 2^31 - 1, runs built to start and end on chunk edges, runs of 2 to 33
  pieces, a padding-id hub of 60,000 contributions, gradients with spread exponents, -0.0 and subnormals, and the
  Reddit-shaped lists of the layer-0 backward.  Gradient rows past ceil(n / group), pad columns and the workspace are
  NaN; the output is a slice of a NaN buffer that must stay NaN around it.  Dropout at p = 0 gives the plain bits.
* gs_embedding_sgd bit for bit at learning rates that are not powers of two, on Node2Vec's two-list call; untouched rows
  and columns >= d hold NaNs with distinct payloads and must come back byte for byte.
* gs_skipgram_grad: aff, neg_aff and gc_pos[:, :d] bit for bit, g, gt, gc_neg and the loss within the derived bounds,
  at B up to 6149 (several pair groups per CTA), S up to 1024, ids outside the tables, duplicates and saturated logits.
* Two calls are bit-identical; the refusals and the empty cases behave as include/graphsage_b200.h says.
The largest bound ratio and RMS statistic per skip-gram output are printed at the end.

tests/test_sparse_grad_numerics_cpu.py shows on a numpy emulation of the kernels that these checks reject subtly wrong
kernels at these shapes."""
import numpy as np
import pytest
import torch

from oracle import sparse_grad as sg

pytestmark = pytest.mark.gpu

NAN_BITS = 0x7FC00000
BAD_IDS = (-1, None, 2 ** 31 - 1)             # None: n_rows
EMBED_D = (1, 31, 32, 33, 127, 128, 129, 256, 602)
GROUPS_SCALES = ((1, 1.0), (10, 0.1), (25, 1.0 / 26), (1, -2.0), (1, 1.0), (10, 1.0), (1, 0.1), (25, -2.0))
EMPTY_LIST = 4
MASKED = (3, 5)                              # the masked lists around the empty one (rate 0.5); the rest mask at 0.25
HUB = 60000


# ---------------------------------------------------------------------------------------------------- inputs
def edge_layout():
    """Sorted ids of a layout whose runs land on chunk edges: runs of 31, 32, 33 and 64 starting at sorted positions
    = 0, 1 and 31 (mod 32), then runs of P = 2, 8, 9, 32 and 33 pieces, single filler ids between them.  Returns
    (ids in ascending order with repeats, the number of ids used: 0 .. n - 1)."""
    seq, nid = [], 0

    def fill_to(res):
        nonlocal nid
        while len(seq) % 32 != res:
            seq.append(nid)
            nid += 1

    for L in (31, 32, 33, 64):
        for res in (0, 1, 31):
            fill_to(res)
            seq += [nid] * L
            nid += 1
    for P in (2, 8, 9, 32, 33):
        fill_to(5)
        seq += [nid] * (27 + 32 * (P - 2) + 7)              # 27 in the first chunk, P - 2 full chunks, 7 in the last
        nid += 1
    return np.array(seq, np.int64), nid


def spread_grad(rs, rows, d, pad_rows=2, pad_cols=3):
    """float32 [rows + pad_rows, d + pad_cols]: Gaussian values times 2^[-30, 30], some -0.0 and subnormals, NaN in
    the rows and columns past [rows, d]."""
    g = np.full((rows + pad_rows, d + pad_cols), np.nan, np.float32)
    v = rs.randn(rows, d) * 2.0 ** rs.randint(-30, 31, size=(rows, d))
    u = rs.rand(rows, d)
    v[u < 0.01] = -0.0
    v[(u >= 0.01) & (u < 0.02)] = rs.randn(int(((u >= 0.01) & (u < 0.02)).sum())) * 2.0 ** -140
    g[:rows, :d] = v
    return g


def embed_case(d, seed=0):
    """Eight lists (ids int32, grad buffer with NaN pads, group, scale) over n_rows = 4000 rows, list 4 empty.  The
    edge layout's ids (the lowest) are split between lists 0 and 1; list 6 holds the padding-id hub (id n_rows - 1)."""
    rs = np.random.RandomState(seed + 17 * d)
    n_rows = 4000
    layout, low = edge_layout()
    owner = rs.randint(0, 2, size=layout.size)
    hub = HUB if d <= 129 else 4000
    sizes = [0, 700, 1203, 555, 0, 999, hub, 4001]
    lists = []
    for l, (group, scale) in enumerate(GROUPS_SCALES):
        ids = rs.randint(low, n_rows - 1, size=sizes[l]).astype(np.int64)
        if l in (0, 1):
            ids = np.concatenate([ids, layout[owner == l]])
        if l == 6:
            ids[rs.rand(ids.size) < 0.9] = n_rows - 1
        if l in (2, 5, 7):
            pos = rs.choice(ids.size, size=9, replace=False)
            ids[pos] = [n_rows if b is None else b for b in BAD_IDS] * 3
        ids = ids[rs.permutation(ids.size)].astype(np.int32)
        if l == EMPTY_LIST:
            ids = ids[:0]
        lists.append((ids, spread_grad(rs, max(-(-ids.size // group), 1), d), group, scale))
    return n_rows, lists


def embed_sites(lists, rate_masked=0.5, rate_rest=0.25):
    return [(1000 + 7 * l, 3 * l + 1, rate_masked if l in MASKED else rate_rest) for l in range(len(lists))]


def reddit_case():
    """test_zz_gpu_identity.test_embedding_grad_full_size's shape: N = 232,965 (+ the padding row), batch 512, fanouts
    25 x 10, d = 64, mean form: 138,752 contributions in four lists."""
    rs = np.random.RandomState(7)
    n_rows, d, B = 232966, 64, 512

    def ids(n):
        x = rs.randint(0, n_rows - 1, size=n)
        x[rs.rand(n) < 0.1] = n_rows - 1
        return x.astype(np.int32)

    lists = []
    for n, k in ((B, 10), (B * 10, 25)):
        lists.append((ids(n), spread_grad(rs, n, d), 1, 1.0))
        lists.append((ids(n * k), spread_grad(rs, n, d), k, 1.0 / k))
    return n_rows, d, lists


def sgd_case(d, seed=0):
    """Node2Vec's context update: lists (batch2, gc_pos) and (negatives, gc_neg), ids shared between them, a long run,
    ids outside the table; table float32 [V, d + 3] with NaNs of distinct payloads everywhere but the touched rows'
    first d columns."""
    rs = np.random.RandomState(seed + d)
    V = 3000
    b2 = rs.randint(0, 400, size=700).astype(np.int32)
    b2[100:500] = 11                                                # a run over many chunks
    neg = rs.choice(400, size=20, replace=False).astype(np.int32)
    b2[::50] = neg[0]
    b2[3], b2[5], neg[7] = -1, V, 2 ** 31 - 1
    lists = [(b2, spread_grad(rs, b2.size, d, pad_cols=1), 1, 1.0), (neg, spread_grad(rs, neg.size, d, pad_cols=1), 1, 1.0)]
    for _, g, _, _ in lists:                                         # keep the update well scaled
        g[np.isfinite(g)] = np.clip(g[np.isfinite(g)], -1e3, 1e3)
    table = (np.arange(V * (d + 3), dtype=np.uint32) % 0x3FFFFF | 0x7FC00000).view(np.float32).reshape(V, d + 3)
    touched = np.unique(np.concatenate([b2, neg]).astype(np.int64))
    touched = touched[(touched >= 0) & (touched < V)]
    table[touched, :d] = rs.randn(touched.size, d).astype(np.float32)
    return table, lists


# (B, S, d): B = 1 .. 2048 keep one pair group per CTA, 2049 and 6149 put several on some CTAs
SG_CASES = [(1, 1, 1), (7, 20, 31), (8, 20, 32), (9, 1, 33), (37, 20, 50), (512, 20, 256), (2048, 20, 33),
            (2049, 20, 50), (6149, 20, 256), (6149, 1, 1), (37, 1024, 31), (512, 1024, 1)]


def sg_case(B, S, d, seed=0):
    """Tables with NaN pads (target [V, d + 3], context [V, d + 3] with the bias in column d), some rows scaled so that
    logits saturate sigma both ways, and pairs / negatives with duplicates and ids outside the tables."""
    rs = np.random.RandomState(seed + 31 * B + 7 * S + d)
    V = 3000
    T = np.full((V, d + 3), np.nan, np.float32)
    C = np.full((V, d + 3), np.nan, np.float32)
    T[:, :d] = rs.uniform(-1, 1, size=(V, d))
    C[:, :d] = rs.randn(V, d) / np.sqrt(d)
    C[:, d] = rs.randn(V) * 0.3
    hot = rs.choice(V, size=V // 20, replace=False)
    T[hot, :d] *= 40.0
    C[hot[:20], d] = rs.choice([-60.0, 60.0], size=20)
    b1, b2 = rs.randint(0, V, size=B).astype(np.int32), rs.randint(0, V, size=B).astype(np.int32)
    neg = rs.choice(V, size=S, replace=S > V).astype(np.int32)
    if B > 5:
        b1[1], b2[2:5] = b1[0], b2[4]
        b2[5] = neg[0]
    bad = np.array([-1, V, 2 ** 31 - 1], np.int32)
    for arr in (b1, b2, neg):
        if arr.size > 3:
            arr[rs.choice(arr.size, size=3, replace=False)] = bad
    if S == 1 and B % 2:
        neg[0] = V                                                   # the only negative outside the table
    return T, C, b1, b2, neg


# ---------------------------------------------------------------------------------------------------- GPU side
MEASURED = {}     # {output: [worst |err| / bound, rms]}


@pytest.fixture(scope="module")
def gs():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    import graphsage_b200
    graphsage_b200._lib.lib()
    yield graphsage_b200
    if MEASURED:
        print("\ngs_skipgram_grad, measured on %s:" % torch.cuda.get_device_name())
        for name, (worst, rms) in sorted(MEASURED.items()):
            print("  %-7s worst |err| / bound = %.3e   rms = %.3e (2^%.1f)"
                  % (name, worst, rms, np.log2(rms) if rms > 0 else -np.inf))


def _nan(*shape):
    return torch.full(shape, float("nan"), dtype=torch.float32, device="cuda")


def _bits(t):
    return t.detach().cpu().contiguous().numpy().view(np.uint32)


def _all_nan(*parts):
    return all(bool((p.reshape(-1).view(torch.int32) == NAN_BITS).all()) for p in parts if p.numel())


def _dev_lists(lists):
    return [(torch.from_numpy(ids).cuda(), torch.from_numpy(g).cuda(), group, scale) for ids, g, group, scale in lists]


def embed_call(gs, lists, n_rows, d, sites=None, ws_bytes=None):
    """The C ABI with a NaN workspace and a NaN buffer around the output: (rc, out [n_rows, d] numpy, surroundings
    all NaN)."""
    ops, lib = gs.ops, gs._lib.lib()
    dl = _dev_lists(lists)
    arr, keep, _ = ops._embed_lists(dl, d, "test")
    nbytes = lib.gs_embedding_grad_workspace_bytes(arr, len(dl), n_rows, d)
    assert nbytes >= 0
    ws = _nan(nbytes // 4 + 1)
    full = _nan(n_rows + 2, d + 9)
    out = full[1:n_rows + 1, 4:4 + d]
    nb = nbytes if ws_bytes is None else ws_bytes
    if sites is None:
        rc = lib.gs_embedding_grad(arr, len(dl), n_rows, d, ops.ptr(out), d + 9, ops.ptr(ws), nb, ops.stream_ptr())
    else:
        c_sites = (gs._lib.DropoutSite * max(len(sites), 1))(*[ops.dropout_site(s) for s in sites])
        rc = lib.gs_embedding_grad_dropout(arr, c_sites, len(dl), n_rows, d, ops.ptr(out), d + 9, ops.ptr(ws), nb,
                                           ops.stream_ptr())
    torch.cuda.synchronize()
    rest = _all_nan(full[0], full[-1], full[1:-1, :4], full[1:-1, 4 + d:])
    return rc, out.cpu().numpy(), rest


def _assert_bits(got, want, what):
    g, w = np.ascontiguousarray(got, np.float32).view(np.uint32), np.ascontiguousarray(want, np.float32).view(np.uint32)
    if not np.array_equal(g, w):
        bad = np.argwhere(g != w)
        i = tuple(bad[0])
        pytest.fail("%s: %d elements differ, first %s: got %r want %r"
                    % (what, bad.shape[0], list(i), float(np.asarray(got)[i]), float(np.asarray(want)[i])))


@pytest.mark.parametrize("d", EMBED_D)
def test_embedding_grad_bit_for_bit(gs, d):
    n_rows, lists = embed_case(d)
    want = sg.embedding_grad_reference(lists, n_rows, d)
    rc, got, rest = embed_call(gs, lists, n_rows, d)
    assert rc == 0 and rest, "wrote outside the output slice"
    _assert_bits(got, want, "gs_embedding_grad d=%d" % d)
    _, again, _ = embed_call(gs, lists, n_rows, d)
    _assert_bits(again, got, "a second call")


@pytest.mark.parametrize("d", EMBED_D)
def test_embedding_grad_dropout_bit_for_bit(gs, d):
    n_rows, lists = embed_case(d, seed=1)
    sites = embed_sites(lists)
    want = sg.embedding_grad_reference(lists, n_rows, d, sites)
    rc, got, rest = embed_call(gs, lists, n_rows, d, sites)
    assert rc == 0 and rest
    _assert_bits(got, want, "gs_embedding_grad_dropout d=%d" % d)
    _, again, _ = embed_call(gs, lists, n_rows, d, sites)
    _assert_bits(again, got, "a second call")
    # p = 0 everywhere: the plain kernel's bits
    zero = [(s, c, 0.0) for s, c, _ in sites]
    _, plain, _ = embed_call(gs, lists, n_rows, d)
    _, masked0, _ = embed_call(gs, lists, n_rows, d, zero)
    _assert_bits(masked0, plain, "dropout at p = 0")


def test_embedding_grad_reddit_shape(gs):
    n_rows, d, lists = reddit_case()
    assert sum(ids.size for ids, _, _, _ in lists) == 138752
    rc, got, rest = embed_call(gs, lists, n_rows, d)
    assert rc == 0 and rest
    _assert_bits(got, sg.embedding_grad_reference(lists, n_rows, d), "Reddit shape")
    sites = [(5, l, 0.5) for l in range(4)]
    rc, got, rest = embed_call(gs, lists, n_rows, d, sites)
    assert rc == 0 and rest
    _assert_bits(got, sg.embedding_grad_reference(lists, n_rows, d, sites), "Reddit shape, dropout")


def sgd_call(gs, table, lists, alpha, d):
    ops, lib = gs.ops, gs._lib.lib()
    dl = _dev_lists(lists)
    arr, keep, _ = ops._embed_lists(dl, d, "test")
    nbytes = lib.gs_embedding_grad_workspace_bytes(arr, len(dl), table.shape[0], d)
    ws = _nan(nbytes // 4 + 1)
    t = torch.from_numpy(table.copy()).cuda()
    rc = lib.gs_embedding_sgd(arr, len(dl), table.shape[0], d, alpha, ops.ptr(t), t.stride(0), ops.ptr(ws), nbytes,
                              ops.stream_ptr())
    torch.cuda.synchronize()
    return rc, t.cpu().numpy()


@pytest.mark.parametrize("lr", [0.05, 0.3])
@pytest.mark.parametrize("d", [1, 51, 257])
def test_embedding_sgd_bit_for_bit(gs, d, lr):
    table, lists = sgd_case(d)
    alpha = float(np.float32(-lr))
    want = sg.embedding_sgd_reference(table, lists, alpha, d)
    rc, got = sgd_call(gs, table, lists, alpha, d)
    assert rc == 0
    assert got.tobytes() == want.tobytes() or _assert_bits(got, want, "gs_embedding_sgd d=%d lr=%g" % (d, lr))
    _, again = sgd_call(gs, table, lists, alpha, d)
    assert again.tobytes() == got.tobytes()


def sg_call(gs, T, C, d, b1, b2, neg, ws_bytes=None):
    """The C ABI into NaN buffers (ldgt = d + 5 > d, ldgc = d + 4 > d + 1, a NaN workspace): (rc, outputs as numpy,
    every element around the outputs still NaN)."""
    ops, lib = gs.ops, gs._lib.lib()
    B, S = b1.size, neg.size
    Td, Cd = torch.from_numpy(T).cuda(), torch.from_numpy(C).cuda()
    i1, i2, ineg = (torch.from_numpy(x).cuda() for x in (b1, b2, neg))
    loss, aff, naff = _nan(3), _nan(B + 2), _nan(B * S + 2)
    gt, gcp, gcn = _nan(B, d + 5), _nan(B, d + 4), _nan(S, d + 4)
    nbytes = lib.gs_skipgram_workspace_bytes(B, S, d)
    ws = _nan(nbytes // 4 + 1)
    rc = lib.gs_skipgram_grad(ops.ptr(Td), T.shape[1], ops.ptr(Cd), C.shape[1], T.shape[0], d, ops.ptr(i1), ops.ptr(i2), B,
                              ops.ptr(ineg), S, ops.ptr(loss[1:]), ops.ptr(aff[1:]), ops.ptr(naff[1:]), ops.ptr(gt), d + 5,
                              ops.ptr(gcp), ops.ptr(gcn), d + 4, ops.ptr(ws), nbytes if ws_bytes is None else ws_bytes,
                              ops.stream_ptr())
    torch.cuda.synchronize()
    rest = _all_nan(loss[0], loss[2:], aff[0], aff[-1], naff[0], naff[-1], gt[:, d:], gcp[:, d + 1:], gcn[:, d + 1:])
    got = dict(loss=float(loss[1]), aff=aff[1:B + 1].cpu().numpy(), neg_aff=naff[1:B * S + 1].reshape(B, S).cpu().numpy(),
               gt=gt[:, :d].cpu().numpy(), gc_pos=gcp[:, :d + 1].cpu().numpy(), gc_neg=gcn[:, :d + 1].cpu().numpy())
    return rc, got, rest


@pytest.mark.parametrize("B, S, d", SG_CASES, ids=["B%d_S%d_d%d" % c for c in SG_CASES])
def test_skipgram_against_the_contract(gs, B, S, d):
    T, C, b1, b2, neg = sg_case(B, S, d)
    rc, got, rest = sg_call(gs, T, C, d, b1, b2, neg)
    assert rc == 0 and rest, "wrote outside the outputs"
    fails, stats = sg.check_skipgram(T, C, d, b1, b2, neg, got)
    for name, (worst, rms) in stats.items():
        w, r = MEASURED.get(name, (0.0, 0.0))
        MEASURED[name] = [max(w, worst), max(r, rms)]
    assert not fails, (fails, stats)
    x = (got["aff"] + sg.skipgram_operands(T, C, d, b1, b2, neg)[2]).astype(np.float64)
    if B >= 512:
        assert (x > 20).any() and (x < -20).any()                  # sigma saturates both ways
    _, again, _ = sg_call(gs, T, C, d, b1, b2, neg)
    for k in got:
        assert np.asarray(again[k], np.float32).tobytes() == np.asarray(got[k], np.float32).tobytes(), k


# ---------------------------------------------------------------------------------------------------- refusals, empty
def test_embedding_refusals_and_empty_cases(gs):
    ops, lib = gs.ops, gs._lib.lib()
    n_rows, lists = embed_case(33)
    d = 33
    # no lists: the whole [n_rows, d] block is zeroed, nothing else written, no workspace needed
    assert lib.gs_embedding_grad_workspace_bytes(None, 0, n_rows, d) == 0
    full = _nan(n_rows + 2, d + 9)
    out = full[1:n_rows + 1, 4:4 + d]
    assert lib.gs_embedding_grad(None, 0, n_rows, d, ops.ptr(out), d + 9, None, 0, ops.stream_ptr()) == 0
    torch.cuda.synchronize()
    assert _bits(out).max() == 0 and _all_nan(full[0], full[-1], full[1:-1, :4], full[1:-1, 4 + d:])
    # n_rows = 0 or d = 0: success without touching out or the workspace
    dl = _dev_lists(lists)
    arr, keep, _ = ops._embed_lists(dl, d, "test")
    for nr, dd in ((0, d), (n_rows, 0)):
        assert lib.gs_embedding_grad(arr, len(dl), nr, dd, None, dd, None, 0, ops.stream_ptr()) == 0
        assert lib.gs_embedding_sgd(arr, len(dl), nr, dd, -0.5, None, dd, None, 0, ops.stream_ptr()) == 0
    # no lists for the update: the table is untouched
    table, _ = sgd_case(5)
    rc, got = sgd_call(gs, table, [], -0.5, 5)
    assert rc == 0 and got.tobytes() == table.tobytes()
    # refusals
    rc, _, rest = embed_call(gs, lists, n_rows, d, ws_bytes=1)
    assert rc == -1 and rest
    big = (gs._lib.EmbedGradList * 9)(*arr, arr[0])
    assert lib.gs_embedding_grad_workspace_bytes(big, 9, n_rows, d) == -1
    for field, value in (("group", 0), ("ldg", d - 1), ("n", -1)):
        bad = (gs._lib.EmbedGradList * len(dl))(*arr)
        setattr(bad[1], field, value)
        assert lib.gs_embedding_grad_workspace_bytes(bad, len(dl), n_rows, d) == -1, field
    assert lib.gs_embedding_grad(arr, len(dl), n_rows, d, ops.ptr(out), d - 1, None, 0, ops.stream_ptr()) == -1
    sites = (gs._lib.DropoutSite * len(dl))(*[ops.dropout_site(s) for s in embed_sites(lists)])
    sites[2].rate = 1.0
    assert lib.gs_embedding_grad_dropout(arr, sites, len(dl), n_rows, d, ops.ptr(out), d + 9, None, 0,
                                         ops.stream_ptr()) == -1
    for alpha in (float("inf"), float("nan")):
        assert lib.gs_embedding_sgd(arr, len(dl), n_rows, d, alpha, ops.ptr(out), d + 9, None, 0, ops.stream_ptr()) == -1
    assert "alpha" in lib.gs_last_error_string().decode()
    torch.cuda.synchronize()
    assert _bits(out).max() == 0                                    # the refused calls wrote nothing


def test_skipgram_refusals(gs):
    lib = gs._lib.lib()
    for B, S, d in ((0, 1, 1), (1, 0, 1), (1, 1, 0), (1, 1025, 1)):
        if S <= 1024:
            assert lib.gs_skipgram_workspace_bytes(B, S, d) == -1
    T, C, b1, b2, neg = sg_case(9, 20, 33)
    d = 33
    rc, _, rest = sg_call(gs, T, C, d, b1, b2, neg, ws_bytes=16)
    assert rc == -1 and rest
    rc, _, rest = sg_call(gs, T, C[:, :d + 1].copy(), d + 1, b1, b2, neg)        # ldc = d + 1 < (d + 1) + 1
    assert rc == -1 and rest
    rc, _, rest = sg_call(gs, T, C, d, b1, b2, np.zeros(1025, np.int32))
    assert rc == -1 and rest
    rc, _, rest = sg_call(gs, T, C, d, b1[:0], b2[:0], neg)
    assert rc == -1 and rest
