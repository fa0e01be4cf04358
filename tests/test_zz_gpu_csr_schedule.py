"""GPU: the hub / short row schedule of csr_rows.cuh where the rest of the suite never reaches it - hub rows past the
first chunk, hub CTAs that take several items, a short role that wraps, the 256 / 257-entry split, hub slices wholly
past F - on every kernel that runs on it: gs_csr_aggregate (mean, mean_self, max over fp32 V = 4, fp32 V = 1 and
bf16 V = 8; the fp32 sum), gs_csr_aggregate_dropout (the masked means and sum) and both phases of gs_csr_max_backward.
Every output is compared bit for bit with the order-exact oracles, every pad column must be +0, and every case runs
twice with identical bits.

The cases and the Python mirror of csr_grid are in test_csr_schedule_cpu.py, which checks that the mirror's constants
are the header's and that every case reaches its regimes on 114 and 132 SMs; here each case asserts its regimes again
for this GPU's SM count and prints them.  An output row of gs_csr_aggregate depends only on its node (dropout positions
are keyed by node), so the oracle runs over the distinct nodes of `rows` and its rows are expanded on the GPU.  Outputs
start as NaN, so a row that no role computes fails."""
import numpy as np
import pytest
import torch

import test_csr_schedule_cpu as cs
from oracle import full_neighbor as fn
from oracle import full_neighbor_dropout as fd
from oracle import full_neighbor_grad as fg
from test_zz_gpu_full_neighbor import dev, table_of

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def gs():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    import graphsage_b200
    graphsage_b200._lib.lib()
    return graphsage_b200


@pytest.fixture(scope="module")
def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def nan_out(n, pitch):
    return torch.full((n, pitch), float("nan"), device="cuda")


def check(buf, want, F, cnt):
    """buf [n, pitch] (the whole out= buffer): columns < F equal want [n, F] bit for bit, columns F .. pitch - 1 are +0.
    On a mismatch, name the first rows that differ and their entry counts."""
    got = buf.view(torch.int32)
    bad = (got[:, :F] != want.view(torch.int32)).any(1) | (got[:, F:] != 0).any(1)
    n_bad = int(bad.sum())
    if n_bad:
        at = bad.nonzero().flatten()[:6].cpu().numpy()
        pytest.fail("%d of %d rows differ; rows %s with %s entries" % (n_bad, len(bad), at.tolist(),
                                                                        np.asarray(cnt)[at].tolist()))


def expand(want_unique, inv):
    return torch.from_numpy(np.ascontiguousarray(want_unique, np.float32)).cuda()[dev(inv.astype(np.int64))]


def twice(run, n, pitch):
    """Two launches into NaN-filled buffers: the first buffer, after checking the second has the same bits."""
    a, b = nan_out(n, pitch), nan_out(n, pitch)
    run(a)
    run(b)
    assert torch.equal(a.view(torch.int32), b.view(torch.int32)), "two runs differ"
    return a


@pytest.mark.parametrize("op,layout,F,wide", cs.AGG_CASES)
def test_aggregate_on_every_regime(gs, sms, op, layout, F, wide):
    c = cs.aggregate_case(sms, layout, F, wide, F == 602, seed=F)
    print("%s %s F=%d out pitch %d: %s" % (op, layout, F, c["pitch"],
                                            cs.require(c["regime"], dead_slice=wide, counts=cs.aggregate_row_counts(layout)
                                                       | ({cs.BIG} if F == 602 else {600}))))
    src, table = table_of(np.random.RandomState(F + 100), c["n_src"], F, layout)
    indptr, indices, rows = dev(c["indptr"]), dev(c["indices"]), dev(c["rows"])
    uniq, inv = np.unique(c["rows"], return_inverse=True)
    want = expand(fn.csr_aggregate(table, c["indptr"], c["indices"], op, uniq), inv)
    got = twice(lambda out: gs.ops.csr_aggregate(src, indptr, indices, op, rows=rows, out=out), len(rows), c["pitch"])
    check(got, want, F, cs.node_counts(c["indptr"], c["rows"]))


@pytest.mark.parametrize("op,p,layout,F,wide", cs.MASK_CASES)
def test_masked_aggregate_on_every_regime(gs, sms, op, p, layout, F, wide):
    c = cs.aggregate_case(sms, layout, F, wide, False, seed=F + 1)
    print("masked %s p=%g %s F=%d out pitch %d: %s" % (op, p, layout, F, c["pitch"],
                                                       cs.require(c["regime"], dead_slice=wide,
                                                                  counts=cs.aggregate_row_counts(layout))))
    rs = np.random.RandomState(F + 101)
    src, table = table_of(rs, c["n_src"], F, layout)
    n = len(c["indptr"]) - 1
    pos_ids = rs.permutation(n + 1).astype(np.int32)           # a local CSR whose rows are named through pos_ids
    neigh, selfs = (9, 3, p), (9, 4, p)
    uniq, inv = np.unique(c["rows"], return_inverse=True)
    want = expand(fd.csr_aggregate_dropout(table, c["indptr"], c["indices"], op, neigh, selfs,
                                           (c["indptr"] * 3, pos_ids, 12345), uniq), inv)
    indptr, indices, rows = dev(c["indptr"]), dev(c["indices"]), dev(c["rows"])
    pm = (dev(c["indptr"] * 3), dev(pos_ids), 12345)
    got = twice(lambda out: gs.ops.csr_aggregate(src, indptr, indices, op, rows=rows, out=out,
                                                 dropout=(neigh, selfs, pm)), len(rows), c["pitch"])
    check(got, want, F, cs.node_counts(c["indptr"], c["rows"]))


def _sum_case(sms, layout, F, wide, with_self):
    c = cs.sum_case(sms, layout, F, wide, with_self, seed=F + 2)
    extra = 1 if with_self else 0
    what = cs.require(c["regime"], dead_slice=wide, counts={d + extra for d in cs.IN_DEGREES})
    assert np.diff(c["t_indptr"])[-1] > cs.LONG                          # the dummy row N is a hub
    return c, what


@pytest.mark.parametrize("layout,F,wide", cs.SUM_CASES)
def test_sum_on_every_regime(gs, sms, layout, F, wide):
    c, what = _sum_case(sms, layout, F, wide, False)
    print("sum %s F=%d out pitch %d: %s; without rows: %s" % (layout, F, c["pitch"], what, cs.describe(c["natural"])))
    n = len(c["t_indptr"]) - 1
    src, x = table_of(np.random.RandomState(F + 102), n, F, layout)
    want_all = fg.csr_sum(x, c["t_indptr"], c["t_indices"])
    t_indptr, t_indices, rows = dev(c["t_indptr"]), dev(c["t_indices"].astype(np.int32)), dev(c["rows"])
    t_cnt = np.diff(c["t_indptr"])
    got = twice(lambda out: gs.ops.csr_aggregate(src, t_indptr, t_indices, "sum", out=out), n, c["pitch"])
    check(got, torch.from_numpy(want_all).cuda(), F, t_cnt)               # the transpose's own rows, as training runs it
    got = twice(lambda out: gs.ops.csr_aggregate(src, t_indptr, t_indices, "sum", rows=rows, out=out), len(rows),
                c["pitch"])
    check(got, torch.from_numpy(want_all).cuda()[rows.long()], F, t_cnt[c["rows"]])


@pytest.mark.parametrize("with_self,layout,F,wide", cs.MASKED_SUM_CASES)
def test_masked_sum_on_every_regime(gs, sms, with_self, layout, F, wide):
    c, what = _sum_case(sms, layout, F, wide, with_self)
    print("masked sum with_self=%s %s F=%d out pitch %d: %s" % (with_self, layout, F, c["pitch"], what))
    n = len(c["t_indptr"]) - 1
    rs = np.random.RandomState(F + 103)
    src, x = table_of(rs, n, F, layout)
    nnz = len(c["indices"])
    pos_map = (c["indptr"] * 3, rs.permutation(n).astype(np.int32), 12345) if with_self else (c["indptr"], None, nnz)
    neigh, selfs = (4, 5, 0.5), (4, 6, 0.3)
    want_all = torch.from_numpy(fd.csr_sum_dropout(x, c["t_indptr"], c["t_indices"], c["t_slot"], neigh, selfs,
                                                   pos_map)).cuda()
    t_indptr, t_indices, rows = dev(c["t_indptr"]), dev(c["t_indices"].astype(np.int32)), dev(c["rows"])
    t_slot = dev(c["t_slot"].astype(np.int32))
    pm = (dev(pos_map[0]), None if pos_map[1] is None else dev(pos_map[1]), pos_map[2])
    t_cnt = np.diff(c["t_indptr"])
    for r, want, cnt in ((None, want_all, t_cnt), (rows, want_all[rows.long()], t_cnt[c["rows"]])):
        got = twice(lambda out: gs.ops.csr_aggregate(src, t_indptr, t_indices, "sum", rows=r, out=out, t_slot=t_slot,
                                                     dropout=(neigh, selfs, pm)), len(want), c["pitch"])
        check(got, want, F, cnt)


def test_max_backward_on_every_regime(gs, sms):
    F = cs.BWD_F
    c = cs.backward_case(sms, seed=5)
    print("max backward F=%d phase (a): %s" % (F, cs.require(c["regime_a"], counts=set(cs.HUB_DEGREES) | {1, 256})))
    print("max backward F=%d phase (b): %s" % (F, cs.require(c["regime_b"], counts=set(cs.IN_DEGREES))))
    assert np.diff(c["t_indptr"])[-1] > cs.LONG                          # the dummy row's transposed row is a hub
    n = len(c["eptr"]) - 1
    rs = np.random.RandomState(6)
    z = rs.randint(0, 4, size=(n, F)).astype(np.float32)                 # four values: ties everywhere, zeros masked
    m = cs.row_max(z, c["eptr"], c["eidx"])
    dm = rs.randn(n, F).astype(np.float32)
    want_s, want_dz = cs.max_backward(z, m, dm, c["eptr"], c["eidx"], c["t_indptr"], c["t_indices"])
    indptr, indices = dev(c["indptr"]), dev(c["indices"])
    t_indptr, t_indices = gs.ops.csr_transpose(indptr, indices)
    E = int(c["t_indptr"][-1])
    assert np.array_equal(t_indptr.cpu().numpy(), c["t_indptr"])
    assert np.array_equal(t_indices[:E].cpu().numpy(), c["t_indices"])
    zd, md, dmd = dev(z), dev(m), dev(dm)
    runs = []
    for _ in range(2):
        s, dz = nan_out(n, F + 3), nan_out(n, F + 5)
        gs.ops.csr_max_backward(zd, md, dmd, indptr, indices, t_indptr, t_indices, s=s, out=dz)
        runs.append((s, dz))
    for buf, want, cnt in ((runs[0][0], want_s, np.diff(c["eptr"])), (runs[0][1], want_dz, np.diff(c["t_indptr"]))):
        check(buf[:, :F], torch.from_numpy(want).cuda(), F, cnt)
        assert buf[:, F:].isnan().all()                                  # nothing is written past F
    for a, b in zip(runs[0], runs[1]):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32)), "two runs differ"
