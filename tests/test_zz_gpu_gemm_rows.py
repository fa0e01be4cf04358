"""GPU: the GEMM part whose A rows are read by id from a table (gs_sage_gemm_rows, ops.TableRows) and the mean layer 0 built
on it, against the gathered-copy path they replace - bit for bit.

* gs_sage_gemm_rows in every math mode equals gs_sage_gemm on the rows gathered into a dense operand: repeated ids, the
  dummy id, ids outside the table, uncovered rows, empty ranges, odd and unaligned row strides, one-shot and prepacked.
* gs_gather_mean without out_self (the self row is no longer fetched) gives the means it gave with out_self.
* MeanAggregator's layer 0 and a whole forward() on the bench shape equal the path with a gathered self-row copy."""
import numpy as np
import pytest
import torch

from oracle import numerics as nu

pytestmark = pytest.mark.gpu

MODES = ["fp32", "tf32x3", "tf32", "bf16"]
MATH = {"fp32": "MATH_FP32_SIMT", "tf32x3": "MATH_TF32X3", "tf32": "MATH_TF32", "bf16": "MATH_BF16"}


@pytest.fixture(scope="module")
def gs():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    import graphsage_b200
    graphsage_b200._lib.lib()
    return graphsage_b200


def _table(rs, n, F, layout):
    """[n + 1, F] fp32 view (last row zero: the dummy row) with the storage layout asked for; NaN outside the view."""
    x = rs.randn(n + 1, F).astype(np.float32)
    x[n] = 0.0
    pitch = {"padded": (F + 7) // 8 * 8, "odd": F + 1 if F % 2 == 0 else F + 2, "offset": (F + 8) // 8 * 8}[layout]
    store = torch.full((n + 1, pitch), float("nan"), device="cuda")
    view = store[:, 1:1 + F] if layout == "offset" else store[:, :F]
    view.copy_(torch.from_numpy(x).cuda())
    return view


def _dense(table, ranges, M):
    """The operand TableRows stands for, materialised with torch indexing (the reference, not the product path)."""
    n = table.shape[0]
    out = torch.zeros((M, table.shape[1]), dtype=torch.float32, device="cuda")
    for ids, row0 in ranges:
        ids = ids.long()
        ids = torch.where((ids < 0) | (ids >= n), torch.full_like(ids, n - 1), ids)
        m = min(ids.numel(), max(M - row0, 0))
        out[row0:row0 + m] = table[ids[:m]]
    return out


CASES = [
    # (M, F, part-0 N, part-1 N, combine, layout, ranges as (row0, n))
    (5632, 602, 128, 128, "concat", "padded", [(0, 512), (512, 5120)]),     # the bench's layer 0
    (300, 37, 50, 50, "add", "odd", [(0, 100), (100, 0), (100, 200)]),       # odd lda, an empty range
    (129, 64, 200, 7, "concat", "offset", [(10, 60), (90, 39)]),            # unaligned A, rows 0-9 and 70-89 uncovered
    (65, 33, 3, 127, "concat", "padded", [(0, 80)]),                         # a range longer than M
]


@pytest.mark.parametrize("math", MODES)
@pytest.mark.parametrize("case", range(len(CASES)))
def test_gemm_rows_by_id_equal_gathered_rows(gs, case, math):
    M, F, N0, N1, combine, layout, spans = CASES[case]
    rs = np.random.RandomState(case * 11 + len(math))
    n = 1000
    table = _table(rs, n, F, layout)
    ranges = []
    for row0, cnt in spans:
        ids = rs.randint(0, n, size=cnt).astype(np.int32)
        if cnt >= 8:                                   # repeats, the dummy id, ids below and above the table
            ids[1] = ids[0]
            ids[2], ids[3], ids[4], ids[5] = n, -1, n + 7, 2**31 - 1
        ranges.append((torch.from_numpy(ids).cuda(), row0))
    xm = torch.from_numpy(rs.randn(M, F).astype(np.float32)).cuda()
    W0 = torch.from_numpy((rs.randn(F, N0) / np.sqrt(F)).astype(np.float32)).cuda()
    W1 = torch.from_numpy((rs.randn(F, N1) / np.sqrt(F)).astype(np.float32)).cuda()
    kw = dict(combine=gs.ops.COMBINE_CONCAT if combine == "concat" else gs.ops.COMBINE_ADD,
              bias=torch.from_numpy(rs.randn(N0 + N1 if combine == "concat" else N0).astype(np.float32)).cuda(),
              act=gs.ops.ACT_RELU, math=getattr(gs.ops, MATH[math]))
    by_id = gs.ops.TableRows(table, ranges, M)
    xs = _dense(table, ranges, M)
    for packed in (None, gs.ops.PackedWeights()):
        for swap in (False, True):                     # the id-read operand as part 0, then as part 1
            if swap and combine == "add" and N0 != N1:
                continue
            got = gs.ops.sage_gemm([(xm, F, W0), (by_id, F, W1)] if swap else [(by_id, F, W0), (xm, F, W1)],
                                   packed=packed, **kw)
            want = gs.ops.sage_gemm([(xm, F, W0), (xs, F, W1)] if swap else [(xs, F, W0), (xm, F, W1)],
                                    packed=gs.ops.PackedWeights() if packed is not None else None, **kw)
            torch.cuda.synchronize()
            assert nu.bits_equal(got.cpu().numpy(), want.cpu().numpy()), (math, CASES[case], swap, packed is not None)


def test_gemm_rows_rejects_bad_ranges(gs):
    table = torch.zeros((10, 8), device="cuda")
    ids = torch.zeros((4,), dtype=torch.int32, device="cuda")
    W = torch.zeros((8, 4), device="cuda")
    with pytest.raises(ValueError):
        gs.ops.TableRows(table, [(ids, 0)] * 5, 4)
    bad = gs.ops.TableRows(table, [(ids, 0)], 4)
    bad.ranges[0] = (ids, -1)                          # a negative first row is refused by the library
    with pytest.raises(RuntimeError):
        gs.ops.sage_gemm([(bad, 8, W)], math=gs.ops.MATH_FP32_SIMT)


def test_gather_mean_without_self_rows_unchanged(gs):
    """The bulk-copy gather skips the self row when nothing reads it; the means must not move by a bit.  Repeated ids, the
    dummy id, ids outside the table, an empty segment and an odd pitch (scalar kernel) are in the mix."""
    rs = np.random.RandomState(5)
    n = 800
    for F, layout in ((602, "padded"), (37, "odd"), (8, "padded")):
        table = _table(rs, n, F, layout)
        segs = []
        row0 = 0
        for cnt, k in ((512, 10), (0, 3), (700, 25), (33, 1)):
            sid = rs.randint(0, n, size=max(cnt, 1)).astype(np.int32)
            nid = rs.randint(0, n, size=max(cnt * k, 1)).astype(np.int32)
            if cnt >= 8:
                sid[:4] = [n, -3, n + 5, sid[4]]
                nid[:4] = [n, -3, n + 5, nid[4]]
            segs.append(gs.ops.Seg(cnt, k, self_ids=torch.from_numpy(sid).cuda(), neigh_ids=torch.from_numpy(nid).cuda(),
                                   out_row0=row0))
            row0 += cnt
        xs, with_self = gs.ops.gather_mean(table, segs, want_self=True)
        _, without = gs.ops.gather_mean(table, segs, want_self=False)
        torch.cuda.synchronize()
        assert nu.bits_equal(with_self.cpu().numpy(), without.cpu().numpy()), (F, layout)


def _bench_like_graph(rs, n, F, max_deg):
    adj = rs.randint(0, n, size=(n + 1, max_deg)).astype(np.int32)
    adj[n] = n
    adj[rs.randint(0, n, size=n // 50)] = n                   # some nodes sample only the dummy node
    feats = np.vstack([rs.randn(n, F).astype(np.float32), np.zeros((1, F), np.float32)])
    return adj, feats


class _GatheredCopy(object):
    """Stands in for ops.TableRows: constructing it yields the dense copy of the rows (the operand the gather used to write),
    which sage_gemm multiplies as an ordinary A matrix."""

    def __new__(cls, table, ranges, M):
        return _dense(table, ranges, M)


def _gathered_copy(gs):
    return _GatheredCopy


@pytest.mark.parametrize("math", MODES)
def test_mean_layer0_equals_gathered_self_path(gs, math, monkeypatch):
    rs = np.random.RandomState(17)
    n, F = 3000, 602
    adj, feats = _bench_like_graph(rs, n, F, 128)
    table = torch.zeros((n + 1, gs.ops.pad_cols(F)), device="cuda")
    table[:, :F] = torch.from_numpy(feats).cuda()
    src = table[:, :F]
    gs.set_default_math(math)
    try:
        agg = gs.MeanAggregator(F, 128, concat=True, device="cuda")
    finally:
        gs.set_default_math("fp32")
    s0 = torch.from_numpy(rs.randint(0, n, size=512).astype(np.int32)).cuda()
    s1 = torch.from_numpy(adj[s0.cpu().numpy()][:, :10].reshape(-1)).cuda()
    s2 = torch.from_numpy(adj[s1.cpu().numpy()][:, :25].reshape(-1)).cuda()
    segs = [gs.ops.Seg(512, 10, self_ids=s0, neigh_ids=s1, out_row0=0),
            gs.ops.Seg(5120, 25, self_ids=s1, neigh_ids=s2, out_row0=512)]
    got = agg.aggregate_rows(src, segs).clone()
    xs, xm = gs.ops.gather_mean(src, segs, want_self=True)
    want = gs.ops.sage_gemm([(xs, F, agg.vars["self_weights"]), (xm, F, agg.vars["neigh_weights"])],
                            combine=gs.ops.COMBINE_CONCAT, act=gs.ops.ACT_RELU, math=agg.math)
    monkeypatch.setattr(gs.ops, "TableRows", _gathered_copy(gs))
    copied = agg.aggregate_rows(src, segs)
    torch.cuda.synchronize()
    assert nu.bits_equal(got.cpu().numpy(), want.cpu().numpy()), math
    assert nu.bits_equal(got.cpu().numpy(), copied.cpu().numpy()), math


@pytest.mark.parametrize("math", ["tf32x3", "fp32"])
def test_forward_bench_shape_equals_gathered_self_path(gs, math, monkeypatch):
    """A whole 2-layer forward (batch 512, fanout 25x10, F = 602) with the self rows read by id equals the forward with the
    gathered self-row copy, bit for bit."""
    rs = np.random.RandomState(23)
    n, F = 20000, 602
    adj, feats = _bench_like_graph(rs, n, F, 128)
    table = torch.zeros((n + 1, gs.ops.pad_cols(F)), device="cuda")
    table[:, :F] = torch.from_numpy(feats).cuda()
    adj_dev = torch.from_numpy(adj).cuda()
    seeds = torch.from_numpy(rs.randint(0, n, size=512).astype(np.int32)).cuda()
    gs.set_default_math(math)
    try:
        sampler = gs.UniformNeighborSampler(adj_dev, seed=123)
        infos = [gs.SAGEInfo("node", sampler, 25, 128), gs.SAGEInfo("node", sampler, 10, 128)]
        model = gs.SampleAndAggregate({"batch_size": 512, "dropout": 0.}, table[:, :F], adj_dev, None, infos, concat=True,
                                      aggregator_type="mean", device="cuda")
        got = model.forward(seeds, normalize=True).clone()
        sampler.counter = 0
        monkeypatch.setattr(gs.ops, "TableRows", _gathered_copy(gs))
        want = model.forward(seeds, normalize=True)
        torch.cuda.synchronize()
    finally:
        gs.set_default_math("fp32")
    assert nu.bits_equal(got.cpu().numpy(), want.cpu().numpy()), math
