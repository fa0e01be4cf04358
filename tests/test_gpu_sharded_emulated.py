"""GPU: the node-partitioned gather with several shards emulated on one GPU (tests/shard_emu.py).

Every "remote" shard is an ordinary device allocation, so the owner search, the replica lookup, the locator forms, the
halo staging passes and both sharded gather kernels run with n_shards > 1 on a one-GPU machine.  Each sharded entry point
sums in the order of its dense counterpart, so results are compared bit for bit with the dense-table kernels (themselves
pinned to numpy and the oracle elsewhere), plus an fp64 numpy check of the means.  What no correct kernel reads is NaN in
the emulated shards (pad columns, one guard row per buffer): an addressing or masking error cannot look plausible."""
import ctypes
import re

import numpy as np
import pytest
import torch

from conftest import rel_err
from shard_emu import EmulatedShards

pytestmark = pytest.mark.gpu

N = 3001
_R16 = (N + 15) // 16
LAYOUTS = {
    "unequal3": [0, 1300, 1301, N],                                   # the middle shard owns a single row
    "empty": [0, 700, 700, N],                                        # shard 1 owns nothing
    "sixteen": [min(N, r * _R16) for r in range(16)] + [N],           # GS_MAX_SHARDS
}
# locators of each mode: 0 global ids, 1 gs_translate_ids (replicas), 2 gs_halo_translate (staging)
MODES = {"plain": (False, False), "replicas": (True, False), "halo": (False, True), "halo+replicas": (True, True)}
MARK = 4096.0                                                         # replica marker: no feature value comes close


@pytest.fixture(scope="module")
def gs():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    import graphsage_b200
    graphsage_b200._lib.lib()
    return graphsage_b200


@pytest.fixture
def variant(gs):
    """Restores the default gather variant whatever the test set."""
    yield lambda v: gs._lib.set_tuning("gather_variant", v)
    gs._lib.set_tuning("gather_variant", 2)


def dev(x):
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def features(F, seed=0):
    return np.random.RandomState(seed).randn(N, F).astype(np.float32)


def dense_table(feats):
    """The dense reference: [N+1, pad_cols(F)] with zero pad columns and the zero dummy row N, as its [N+1, F] view."""
    F = feats.shape[1]
    t = torch.zeros((N + 1, (F + 7) // 8 * 8), dtype=torch.float32, device="cuda")
    t[:N, :F] = dev(feats)
    return t[:, :F]


def replica_ids(row_start, my):
    """Remote ids for my shard's replicas: both ids at every even-numbered shard boundary plus random remote ids (the
    other boundaries stay owner-resolved)."""
    lo, hi = row_start[my], row_start[my + 1]
    cand = set(np.random.RandomState(100 + my).randint(0, N, size=150).tolist())
    for r, b in enumerate(row_start):
        if r % 2 == 0:
            cand.update((b - 1, b))
    return np.array(sorted(c for c in cand if 0 <= c < N and not lo <= c < hi), np.int64)


def edge_ids(row_start):
    """Every shard boundary from both sides, the dummy id N and ids outside [0, N]."""
    e = [b for b in row_start] + [b - 1 for b in row_start] + [-5, -1, N, N + 3]
    return np.array(e, np.int64)


def id_pool(row_start, n_random=2000, seed=1):
    ids = np.concatenate([np.random.RandomState(seed).randint(0, N, size=n_random), edge_ids(row_start)])
    return np.random.RandomState(seed + 1).permutation(ids).astype(np.int32)


def clamp(ids):
    ids = np.asarray(ids, np.int64)
    return np.where((ids < 0) | (ids >= N), N, ids)


def emulate(feats, row_start, my, mode="plain"):
    rep, halo = MODES[mode]
    return EmulatedShards(feats, row_start, my, replica_ids(row_start, my) if rep else None, stage_halo=halo)


def rule_locators(ids, row_start, my, rep):
    """The documented locator rule, restated: remap[id] when the row is held locally (own row id - lo, the zero row for ids
    outside [0, N), replica i at n_local + 1 + i), otherwise -id - 1."""
    ids = np.asarray(ids, np.int64)
    lo, hi = row_start[my], row_start[my + 1]
    out = -ids - 1
    own = (ids >= lo) & (ids < hi)
    out[own] = ids[own] - lo
    if len(rep):
        pos = np.searchsorted(rep, ids)
        hit = (ids >= 0) & (ids < N) & (pos < len(rep))
        hit[hit] = rep[pos[hit]] == ids[hit]
        out[hit] = (hi - lo) + 1 + pos[hit]
    out[(ids < 0) | (ids >= N)] = hi - lo
    return out


def full_width(t, pitch):
    """The whole [rows, pitch] buffer behind a [rows, F] view returned by ops.gather_rows."""
    return t.as_strided((t.shape[0], pitch), (t.stride(0), 1))


# ---------------------------------------------------------------- the emulator itself
def test_emulator_layout_and_single_rank_cross_check(gs):
    from graphsage_b200 import parallel
    F = 50
    feats = features(F, 3)
    real = parallel.ShardedFeatures(feats, N)
    emu = EmulatedShards(feats, [0, N], 0)
    for name in ("n_shards", "my_shard", "n_global_rows", "zero_row"):
        assert getattr(emu._table, name) == getattr(real._table, name), name
    assert list(emu._table.row_start[:2]) == list(real._table.row_start[:2]) == [0, N]
    assert emu.remap is None and real.remap is None
    assert (emu.shape, emu.pitch, emu.zero_row, emu.world, emu.rank) == (real.shape, real.pitch, real.zero_row, 1, 0)
    assert torch.equal(emu.local[:N + 1, :F], real.local[:, :F])
    assert bool(torch.isnan(emu.local[:, F:]).all()) and bool(torch.isnan(emu.local[N + 1]).all())
    ids = dev(id_pool([0, N]))
    assert torch.equal(gs.ops.gather_rows(emu, ids), gs.ops.gather_rows(real, ids))
    seg = [gs.ops.Seg(40, 13, self_ids=ids[:40], neigh_ids=ids[40:40 + 520])]
    a, b = gs.ops.gather_mean(emu, seg, include_self=True), gs.ops.gather_mean(real, seg, include_self=True)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    real.close()
    emu.close()
    # multi-shard layout and the replica remap against the rule, for every shard of every layout
    for row_start in LAYOUTS.values():
        for my in range(len(row_start) - 1):
            emu = emulate(feats, row_start, my, "replicas")
            lo, hi = row_start[my], row_start[my + 1]
            rep = emu.replica_ids
            every = np.arange(N + 1)
            assert np.array_equal(emu.remap.cpu().numpy(), np.where(rule_locators(every, row_start, my, rep) < 0, -1,
                                                                    rule_locators(every, row_start, my, rep)))
            for r, buf in enumerate(emu.buffers):
                n_rows = row_start[r + 1] - row_start[r] + (1 + len(rep) if r == my else 0)
                assert buf.shape == (n_rows + 1, emu.pitch) and buf.data_ptr() % 16 == 0
                assert bool(torch.isnan(buf[:, F:]).all()) and bool(torch.isnan(buf[-1]).all())
            assert bool((emu.local[hi - lo, :F] == 0).all())
            assert torch.equal(emu.replica_rows(), dev(feats[rep]))
            emu.close()


# ---------------------------------------------------------------- gs_gather_rows_sharded
@pytest.mark.parametrize("F", [602, 50, 1500])
@pytest.mark.parametrize("mode", ["plain", "replicas"])
@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_gather_rows_emulated(gs, layout, mode, F):
    row_start = LAYOUTS[layout]
    feats = features(F)
    dense = dense_table(feats)
    ids_np = id_pool(row_start)
    ids = dev(ids_np)
    want = dense[dev(clamp(ids_np))]
    for my in range(len(row_start) - 1):
        emu = emulate(feats, row_start, my, mode)
        out = gs.ops.gather_rows(emu, ids)
        assert torch.equal(out, want), (layout, mode, F, my)
        assert bool((full_width(out, emu.pitch)[:, F:] == 0).all())
        emu.close()


@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_replica_rows_are_read(gs, layout, variant):
    """Replica rows hold their owners' values, so parity alone cannot tell the replica branch from the owner branch: mark
    the replica rows of my shard's buffer and require the marker for replicated ids, the owner's values for the rest."""
    row_start = LAYOUTS[layout]
    F = 602
    feats = features(F, 5)
    dense = dense_table(feats)
    ids_np = id_pool(row_start, n_random=1400)
    ids = dev(ids_np)
    k = 13
    n = len(ids_np) // (k + 1)
    for my in range(len(row_start) - 1):
        for mode in ("replicas", "halo+replicas"):
            emu = emulate(feats, row_start, my, mode)
            rep = emu.replica_ids
            assert len(rep) and np.isin(rep, ids_np).any()
            emu.replica_rows().fill_(MARK)
            marked = dense.clone()
            marked[dev(rep)] = MARK
            want = marked[dev(clamp(ids_np))]
            out = gs.ops.gather_rows(emu, ids)
            assert torch.equal(out, want), (layout, my, mode)
            assert bool((out[torch.from_numpy(np.isin(ids_np, rep)).cuda()] == MARK).all())
            seg = [gs.ops.Seg(n, k, self_ids=ids[:n], neigh_ids=ids[n:n + n * k])]
            for v in (2, 0):
                variant(v)
                a = gs.ops.gather_mean(emu, seg, include_self=True)
                b = gs.ops.gather_mean(marked, seg, include_self=True)
                assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]), (layout, my, mode, v)
            variant(2)
            emu.close()


# ---------------------------------------------------------------- gs_translate_ids
@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_translate_ids_emulated(gs, layout):
    row_start = LAYOUTS[layout]
    feats = features(8)
    ids_np = id_pool(row_start)
    for my in range(len(row_start) - 1):
        emu = emulate(feats, row_start, my, "replicas")
        got = gs.ops.translate_ids(emu, dev(ids_np)).cpu().numpy()
        assert np.array_equal(got, rule_locators(ids_np, row_start, my, emu.replica_ids)), (layout, my)
        emu.close()


# ---------------------------------------------------------------- halo staging: begin -> claim -> fetch -> translate
def halo_stage(gs, emu, lists):
    """The staging passes in the order ops._shard_prepare issues them; returns (count, stage_ids, staging, locators)."""
    lib, ptr, check, stream = gs._lib.lib(), gs._lib.ptr, gs._lib.check, gs._lib.stream_ptr()
    capacity = sum(t.numel() for t in lists)
    claim = torch.empty((N + 1,), dtype=torch.int32, device="cuda")
    count = torch.empty((1,), dtype=torch.int32, device="cuda")
    stage_ids = torch.full((capacity,), -7, dtype=torch.int32, device="cuda")
    staging = torch.full((capacity, emu.pitch), float("nan"), dtype=torch.float32, device="cuda")
    check(lib.gs_halo_begin(ptr(claim), N + 1, ptr(count), stream))
    for t in lists:
        check(lib.gs_halo_claim(emu.c_table(), ptr(t), t.numel(), ptr(claim), ptr(count), ptr(stage_ids), capacity, stream))
    check(lib.gs_halo_fetch(emu.c_table(), emu.shape[1], emu.pitch, ptr(stage_ids), ptr(count), capacity, ptr(staging),
                            emu.pitch, stream))
    locs = []
    for t in lists:
        locs.append(torch.empty_like(t))
        check(lib.gs_halo_translate(emu.c_table(), ptr(t), t.numel(), ptr(claim), ptr(locs[-1]), stream))
    torch.cuda.synchronize()
    return int(count.item()), stage_ids.cpu().numpy(), staging, [x.cpu().numpy() for x in locs]


@pytest.mark.parametrize("F", [602, 50])
@pytest.mark.parametrize("mode", ["plain", "replicas"])
@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_halo_staging_emulated(gs, layout, mode, F):
    row_start = LAYOUTS[layout]
    feats = features(F, 7)
    dense = dense_table(feats)
    pool = id_pool(row_start, n_random=900)
    self_np = pool[:300]
    # the neighbour list repeats every self id, repeats itself, and the third list is the first one again (its own tensor)
    neigh_np = np.random.RandomState(8).permutation(np.concatenate([self_np, pool, pool[::3]])).astype(np.int32)
    lists_np = [self_np, neigh_np, self_np.copy()]
    every = np.concatenate(lists_np)
    for my in range(len(row_start) - 1):
        emu = emulate(feats, row_start, my, mode)
        rule = [rule_locators(x, row_start, my, emu.replica_ids) for x in lists_np]
        remote = set(every[np.concatenate(rule) < 0].tolist())
        count, stage_ids, staging, locs = halo_stage(gs, emu, [dev(x) for x in lists_np])
        assert count == len(remote), (layout, mode, my)
        staged = stage_ids[:count]
        assert len(set(staged.tolist())) == count and set(staged.tolist()) == remote
        assert bool((stage_ids[count:] == -7).all())
        assert torch.equal(staging[:count, :F], dense[dev(staged.astype(np.int64))])
        for ids, want, got in zip(lists_np, rule, locs):
            local = want >= 0
            assert np.array_equal(got[local], want[local])
            slot = -got[~local].astype(np.int64) - 1
            assert ((slot >= 0) & (slot < count)).all() and np.array_equal(staged[slot], ids[~local])
        emu.close()


# ---------------------------------------------------------------- gs_gather_mean_sharded (both kernels)
SEGS_MIX = [(40, 25), (0, 13), (9, 128), (17, 14)]          # (n, k): four segments, one of them empty
SEGS_SMALL_K = [(33, 1), (21, 13)]


def id_segments(gs, pool, spec, seed):
    rs = np.random.RandomState(seed)
    segs, row = [], 0
    for n, k in spec:
        s = dev(rs.choice(pool, size=n).astype(np.int32))
        nb = dev(rs.choice(pool, size=n * k).astype(np.int32))
        segs.append(gs.ops.Seg(n, k, self_ids=s, neigh_ids=nb, out_row0=row))
        row += n
    return segs


def range_segments(gs):
    """Dense-range addressing (self_row0 / neigh_row0, no ids) across shard boundaries and past the last row."""
    return [gs.ops.Seg(100, 14, self_row0=1250, neigh_row0=600), gs.ops.Seg(8, 13, self_row0=2990, neigh_row0=2900, out_row0=100)]


def fp64_means(feats, segs, include_self):
    t = np.vstack([feats, np.zeros((1, feats.shape[1]), np.float32)]).astype(np.float64)
    out = []
    for s in segs:
        self_ids = s.self_ids.cpu().numpy() if s.self_ids is not None else s.self_row0 + np.arange(s.n)
        neigh = s.neigh_ids.cpu().numpy() if s.neigh_ids is not None else s.neigh_row0 + np.arange(s.n * s.k)
        rows = t[clamp(neigh)].reshape(s.n, s.k, t.shape[1])
        if include_self:
            rows = np.concatenate([rows, t[clamp(self_ids)][:, None]], axis=1)
        out.append(rows.mean(axis=1))
    return np.vstack(out)


@pytest.mark.parametrize("gv", [2, 0])
@pytest.mark.parametrize("F", [602, 50, 1500])
@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_gather_mean_emulated(gs, layout, F, gv, variant):
    row_start = LAYOUTS[layout]
    feats = features(F, 11)
    dense = dense_table(feats)
    pool = id_pool(row_start)
    calls = [id_segments(gs, pool, SEGS_MIX, 12), id_segments(gs, pool, SEGS_SMALL_K, 13), range_segments(gs)]
    variant(gv)
    flags = [(False, True), (True, False), (False, False), (True, True)]     # (include_self, want_self)
    refs = {}
    for ci, segs in enumerate(calls):
        for inc, ws in flags:
            refs[ci, inc, ws] = gs.ops.gather_mean(dense, segs, include_self=inc, want_self=ws)
        for inc in (False, True):
            xm = refs[ci, inc, True][1][:, :F].cpu().numpy()
            assert rel_err(xm, fp64_means(feats, segs, inc)) < 1e-6, (ci, inc)
    for my in range(len(row_start) - 1):
        for mode in MODES:
            emu = emulate(feats, row_start, my, mode)
            for ci, segs in enumerate(calls):
                for inc, ws in flags:
                    xs, xm = gs.ops.gather_mean(emu, segs, include_self=inc, want_self=ws)
                    rs_, rm = refs[ci, inc, ws]
                    assert torch.equal(xm, rm), (layout, F, gv, my, mode, ci, inc, ws)
                    assert (xs is None) == (not ws) and (xs is None or torch.equal(xs, rs_))
            emu.close()


def test_sharded_gather_mean_refuses_mixed_addressing(gs):
    """With replicas or halo staging the id lists are translated to locators, which a row-range segment cannot carry: a
    call that mixes both forms must be refused (before, the replica form read its row ranges as local row indices)."""
    row_start = LAYOUTS["unequal3"]
    feats = features(50, 14)
    dense = dense_table(feats)
    segs = id_segments(gs, id_pool(row_start), [(20, 5)], 15) + [gs.ops.Seg(10, 4, self_row0=1290, neigh_row0=1280, out_row0=20)]
    ref = gs.ops.gather_mean(dense, segs)
    for mode in MODES:
        emu = emulate(feats, row_start, 0, mode)
        if mode == "plain":                                  # global ids and row ranges address the same rows
            got = gs.ops.gather_mean(emu, segs)
            assert torch.equal(got[0], ref[0]) and torch.equal(got[1], ref[1])
        else:
            with pytest.raises(ValueError, match="by ids"):
                gs.ops.gather_mean(emu, segs)
        emu.close()


# ---------------------------------------------------------------- refusals: errors, not launches
def test_sharded_entry_points_refuse_bad_shard_tables(gs):
    lib, ptr, check, stream = gs._lib.lib(), gs._lib.ptr, gs._lib.check, gs._lib.stream_ptr()
    F = 50
    row_start = LAYOUTS["unequal3"]
    emu = emulate(features(F), row_start, 1, "replicas")
    pitch = emu.pitch
    ids = dev(id_pool(row_start, n_random=60))
    n = ids.numel()
    out = torch.full((n, pitch), -7.0, device="cuda")
    claim = torch.full((N + 1,), -1, dtype=torch.int32, device="cuda")
    count = torch.zeros((1,), dtype=torch.int32, device="cuda")
    stage_ids = torch.full((n,), -7, dtype=torch.int32, device="cuda")
    staging = torch.full((n, pitch), -7.0, device="cuda")
    locs = torch.full((n,), -7, dtype=torch.int32, device="cuda")
    seg = gs.ops.Seg(4, 13, self_ids=ids[:4], neigh_ids=ids[4:56])
    arr = (gs._lib.Segment * 1)(seg.c_struct())

    def entries(t, locators=0, staging_ptr=None):
        return {
            "gs_gather_rows_sharded": lambda: lib.gs_gather_rows_sharded(t, gs._lib.GS_F32, F, pitch, ptr(ids), n, ptr(out), pitch,
                                                                         stream),
            "gs_gather_mean_sharded": lambda: lib.gs_gather_mean_sharded(t, gs._lib.GS_F32, F, pitch, arr, 1, 0, locators,
                                                                         staging_ptr, ptr(out), ptr(out), pitch, stream),
            "gs_halo_claim": lambda: lib.gs_halo_claim(t, ptr(ids), n, ptr(claim), ptr(count), ptr(stage_ids), n, stream),
            "gs_halo_translate": lambda: lib.gs_halo_translate(t, ptr(ids), n, ptr(claim), ptr(locs), stream),
            "gs_halo_fetch": lambda: lib.gs_halo_fetch(t, F, pitch, ptr(stage_ids), ptr(count), n, ptr(staging), pitch, stream),
        }

    def altered(**kw):
        t = emu.table_copy()
        for key, v in kw.items():
            if key == "row_start":
                for i, x in enumerate(v):
                    t.row_start[i] = x
            elif key == "misalign":
                t.base[v] = t.base[v] + 4
            else:
                setattr(t, key, v)
        return t

    cases = [
        (altered(row_start=[0, 1300, 1301, N - 1]), "row_start must run from 0 to n_global_rows - 1"),
        (altered(row_start=[0, 1300, 1200, N]), "row_start must be non-decreasing (shard 1)"),
        (altered(n_shards=0), "n_shards=0 (max 16)"),
        (altered(n_shards=17), "n_shards=17 (max 16)"),
        (altered(my_shard=3), "my_shard=3"),
        (altered(my_shard=-1), "my_shard=-1"),
        (altered(misalign=2), "shard 2 pointer NULL or not 16-byte aligned"),
    ]
    for t, msg in cases:
        for name, call in entries(ctypes.byref(t)).items():
            with pytest.raises(RuntimeError, match=re.escape("%s: %s" % (name, msg))):
                check(call())
    with pytest.raises(RuntimeError, match=re.escape("gs_gather_mean_sharded: ids_are_locators = 2 needs the staging buffer")):
        check(entries(emu.c_table(), locators=2)["gs_gather_mean_sharded"]())
    plain = emulate(features(F), row_start, 1, "plain")
    with pytest.raises(RuntimeError, match=re.escape("gs_translate_ids: the table has no remap (no replicas)")):
        gs.ops.translate_ids(plain, ids)
    torch.cuda.synchronize()
    # nothing was launched: every buffer a kernel would have written still holds its sentinel
    assert bool((out == -7).all()) and bool((staging == -7).all()) and bool((stage_ids == -7).all())
    assert bool((locs == -7).all()) and bool((claim == -1).all()) and int(count.item()) == 0
    plain.close()
    emu.close()


# ---------------------------------------------------------------- every sharded entry point launches its own kernel
def test_sharded_kernels_each_recorded_by_profiler(gs, variant):
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    row_start = LAYOUTS["unequal3"]
    F = 602
    feats = features(F, 31)
    pool = id_pool(row_start)
    segs = id_segments(gs, pool, SEGS_MIX, 32)
    emus = {mode: emulate(feats, row_start, 0, mode) for mode in ("plain", "replicas", "halo")}
    ids = dev(pool)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(2):                                  # the first launches of a profiled region can go unrecorded
            gs.ops.gather_rows(emus["plain"], ids)
            gs.ops.translate_ids(emus["replicas"], ids)
            for mode, e in emus.items():
                gs.ops.gather_mean(e, segs)
            variant(0)
            gs.ops.gather_mean(emus["halo"], segs)
            variant(2)
        torch.cuda.synchronize()
    names = sorted(set(e.name for e in prof.events() if e.device_type == DeviceType.CUDA))
    if not names:
        pytest.skip("the profiler recorded no device activity here (CUPTI unavailable)")
    print("\n".join(names))
    for k in ("translate_ids_kernel", "halo_claim_kernel", "halo_fetch_kernel", "halo_translate_kernel",
              "gather_rows_sharded_kernel", "gather_mean_sharded_kernel"):
        assert any(k in nm for nm in names), (k, names)
    assert any("gather_mean_tma2_kernel" in nm and "ShardRows" in nm for nm in names), names
    for e in emus.values():
        e.close()


# ---------------------------------------------------------------- models over the emulated table
def model_inputs(F=602, md=32, B=64, seed=41):
    rs = np.random.RandomState(seed)
    adj = rs.randint(0, N, size=(N + 1, md)).astype(np.int32)
    adj[N] = N
    adj[5] = N                                             # an isolated node: dummy neighbours (the zero row)
    adj[1300, :8] = 1299                                   # the one-row shard and its neighbours across both boundaries
    adj[1301, :8] = 1300
    feats = rs.randn(N, F).astype(np.float32)
    seeds = rs.randint(0, N, size=B).astype(np.int32)
    seeds[:5] = [5, 1299, 1300, 1301, N - 1]
    return adj, feats, seeds


def build_forward_model(gs, table, adj_dev, kind, concat, dim, B):
    gs.inits.manual_seed(7)
    sampler = gs.UniformNeighborSampler(adj_dev, seed=123)
    infos = [gs.SAGEInfo("node", sampler, 25, dim), gs.SAGEInfo("node", sampler, 10, dim)]
    return gs.SampleAndAggregate({"batch_size": B, "dropout": 0.}, table, adj_dev, None, infos, concat=concat,
                                 aggregator_type=kind), sampler


@pytest.mark.parametrize("math", ["fp32", "tf32x3"])
@pytest.mark.parametrize("kind,concat,dim", [("mean", True, 64), ("gcn", False, 64), ("maxpool", True, 32),
                                             ("meanpool", False, 32)])
def test_forward_emulated_vs_dense(gs, kind, concat, dim, math):
    """The two-GPU test's assertion on one GPU: the partitioned forward equals the single-table forward bit for bit."""
    adj, feats, seeds = model_inputs()
    adj_dev, seeds_t = dev(adj), dev(seeds)
    B = len(seeds)
    gs.set_default_math(math)
    try:
        m, _ = build_forward_model(gs, dense_table(feats), adj_dev, kind, concat, dim, B)
        want = m.forward(seeds_t, normalize=True)
        for my in range(3):
            for mode in MODES:
                emu = emulate(feats, LAYOUTS["unequal3"], my, mode)
                m, _ = build_forward_model(gs, emu, adj_dev, kind, concat, dim, B)
                got = m.forward(seeds_t, normalize=True)
                assert torch.equal(got, want), (kind, math, my, mode, float((got - want).abs().max()))
                emu.close()
    finally:
        gs.set_default_math("fp32")


@pytest.mark.parametrize("mode", ["halo", "halo+replicas"])
def test_graphed_forward_emulated_halo(gs, mode):
    """The halo passes allocate per-call buffers; under CUDA-graph capture they live in the graph's pool.  Replays must
    reproduce the eager forwards (and the dense table's)."""
    adj, feats, seeds = model_inputs(F=50)
    adj_dev, seeds_t = dev(adj), dev(seeds)
    B = len(seeds)
    dense_m, _ = build_forward_model(gs, dense_table(feats), adj_dev, "mean", True, 64, B)
    dense0 = dense_m.forward(seeds_t).clone()
    dense1 = dense_m.forward(seeds_t).clone()
    emu = emulate(feats, LAYOUTS["unequal3"], 2, mode)
    m, sampler = build_forward_model(gs, emu, adj_dev, "mean", True, 64, B)
    eager0 = m.forward(seeds_t).clone()
    eager1 = m.forward(seeds_t).clone()
    assert torch.equal(eager0, dense0) and torch.equal(eager1, dense1)
    sampler.counter = 0
    runner = m.graphed(B, normalize=True)
    r0 = runner(seeds_t).clone()
    r1 = runner(seeds_t).clone()
    torch.cuda.synchronize()
    assert torch.equal(r0, eager0) and torch.equal(r1, eager1)
    runner.reset(0)
    assert torch.equal(runner(seeds_t), eager0)
    runner.close()
    emu.close()


def test_unsupervised_train_steps_emulated(gs):
    """Three UnsupervisedGraphsage steps (distributed=False, dropout 0) on emulated shards and on the dense table: the
    losses and every weight after every step are bit-identical."""
    rs = np.random.RandomState(51)
    md, F, B = 16, 32, 48
    adj = rs.randint(0, N, size=(N + 1, md)).astype(np.int32)
    adj[N] = N
    feats = rs.randn(N, F).astype(np.float32)
    deg = rs.randint(1, 30, size=N).astype(np.float64)
    adj_dev = dev(adj)
    batches = []
    for step in range(3):
        b1 = rs.randint(0, N, size=B).astype(np.int32)
        batches.append((torch.from_numpy(b1), torch.from_numpy(adj[b1, step % md].astype(np.int32))))
    gs.set_default_math("fp32")

    def run(table):
        gs.inits.manual_seed(9)
        sampler = gs.UniformNeighborSampler(adj_dev, seed=123)
        infos = [gs.SAGEInfo("node", sampler, 5, 16), gs.SAGEInfo("node", sampler, 3, 16)]
        m = gs.UnsupervisedGraphsage({"batch_size": B, "dropout": 0.}, table, adj_dev, deg, infos, concat=True,
                                     aggregator_type="mean", neg_sample_size=7, learning_rate=0.01, seed=50)
        trace = []
        for b1, b2 in batches:
            loss = m.train_step(b1, b2)
            trace.append((loss.clone(), [p.detach().clone() for p in m.parameters()]))
        return trace

    want = run(dense_table(feats))
    for my, mode in ((0, "plain"), (1, "replicas"), (2, "halo+replicas")):
        emu = emulate(feats, LAYOUTS["unequal3"], my, mode)
        got = run(emu)
        for step, ((la, pa), (lb, pb)) in enumerate(zip(got, want)):
            assert torch.equal(la, lb), (my, mode, step, float(la), float(lb))
            assert all(torch.equal(x, y) for x, y in zip(pa, pb)), (my, mode, step)
        emu.close()
