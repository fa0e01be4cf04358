"""GPU: the CSR transpose, dropout, int8 / bf16 row conversion, staging and R-MAT kernels past one pass of their capped
grids - where the rest of the suite never reaches them.  Every case is sized from this GPU's SM count so that each
grid-stride loop takes three or more passes with a partial last one, and every output is compared bit for bit (byte for
byte for int8 rows) with a vectorised reference that test_grid_stride_regimes_cpu.py checks against the oracle:

  gs_csr_transpose      N + 1 = 2^19 and 2^19 + 1 rows, plain and with t_slot, with and without the self entry: empty
                        rows, an out-degree hub of 10^5 entries, entries -1, N, N + 1 and INT32_MAX
  gs_dropout_apply      F = 1, 5 and 602; group 1 and 25, accumulate, in place, positions above 2^30
  gs_quantize_rows_i8   F = 1, 37, 602 and 1536, every byte of every row; Int8Features quantised in several chunks
  gs_cast_rows_bf16     the vector kernel and the scalar one (odd out_pitch) over random bit patterns and the edge values
  staging               halo claim / fetch / translate over 10^6 ids at F = 602, 1500, 2000 (2112 rows per fetch pass on
                        132 SMs, rows wider than 640 and 1280 columns); gs_translate_ids with replicas; HostFeatures.stage
                        for fp32, bf16 and int8 rows, without a cache and with one filled in several passes; the fetches
                        with *count > capacity
  R-MAT                 gs_rmat_degrees at scale 21, the whole CSR at scale 18 (a row of about 37,000 entries) with no,
                        one and thousands of long rows

Outputs are slices of larger buffers filled with a sentinel (NaN where the type has one), so an element that no thread
writes, or a write past the slice, fails.  Each call runs twice and must give the same bits; the halo and host staging
take their slots by atomics, so there each run is checked on its own - sets and rows, not slot numbers."""
import numpy as np
import pytest
import torch

import test_grid_stride_regimes_cpu as cs
from oracle import int8_rows
from oracle import rmat as ormat
from shard_emu import EmulatedShards

pytestmark = pytest.mark.gpu

LEAD, TRAIL = 3, 5                      # margin rows (or elements) around every output
S32, S64, S8 = -777_777, -(2**40) - 7, 0xA5


@pytest.fixture(scope="module")
def gs():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    import graphsage_b200
    graphsage_b200._lib.lib()
    return graphsage_b200


@pytest.fixture(scope="module")
def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def dev(x):
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def ptr(t):
    return 0 if t is None else t.data_ptr()


def call(gs, name, *args):
    gs._lib.check(getattr(gs._lib.lib(), name)(*args, gs._lib.stream_ptr()))


def bits(a):
    """An array (or a tensor, bf16 included) as unsigned integers of its item size."""
    if torch.is_tensor(a):
        a = (a.view(torch.int16) if a.dtype == torch.bfloat16 else a).cpu().numpy()
    a = np.ascontiguousarray(a)
    return a.view({1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}[a.itemsize])


def same(got, want, what):
    g, w = bits(got), bits(want)
    assert g.shape == w.shape, (what, g.shape, w.shape)
    bad = np.nonzero((g != w).reshape(-1))[0]
    if len(bad):
        pytest.fail("%s: %d of %d elements differ; first at %s: got %s, want %s" % (
            what, len(bad), g.size, bad[:5].tolist(), [hex(x) for x in g.reshape(-1)[bad[:5]].tolist()],
            [hex(x) for x in w.reshape(-1)[bad[:5]].tolist()]))


def framed(shape, fill, dtype):
    """(buffer, view): a buffer of LEAD + shape[0] + TRAIL rows filled with `fill`, and its middle rows."""
    buf = torch.full((LEAD + shape[0] + TRAIL,) + tuple(shape[1:]), fill, dtype=dtype, device="cuda")
    return buf, buf[LEAD:LEAD + shape[0]]


def same_frame(buf, init, region, want, what):
    """buf holds its initial bits `init` everywhere but `region`, and `want` there."""
    e = bits(init).copy()
    e[region] = bits(want)
    same(buf, e, what)


# ---------------------------------------------------------------- gs_csr_transpose
GRAPHS = {}


def transpose_graph(n):
    if n not in GRAPHS:
        GRAPHS[n] = cs.transpose_graph(n, seed=n % 97)
    return GRAPHS[n]


def transpose(gs, d_ptr, d_idx, n, nnz, with_self, slots):
    """gs_csr_transpose into framed sentinel outputs: the whole (t_indptr, t_indices, t_slot or None) buffers."""
    ws_self = int(with_self)
    cap = nnz + (n + 1) * (1 + ws_self)
    nbytes = gs._lib.lib().gs_csr_transpose_workspace_bytes(n, nnz, ws_self)
    assert nbytes > 0
    work = torch.empty((nbytes,), dtype=torch.uint8, device="cuda")
    tp, tpv = framed((n + 2,), S64, torch.int64)
    ti, tiv = framed((cap,), S32, torch.int32)
    ts, tsv = framed((cap,), S32, torch.int32) if slots else (None, None)
    call(gs, "gs_csr_transpose", ptr(d_ptr), ptr(d_idx), n, nnz, ws_self, ptr(tpv), ptr(tiv), ptr(tsv), ptr(work), nbytes)
    return [None if t is None else t.cpu().numpy() for t in (tp, ti, ts)]


@pytest.mark.parametrize("with_self", [False, True])
@pytest.mark.parametrize("n", cs.TRANSPOSE_NS)
def test_csr_transpose_on_every_regime(gs, sms, n, with_self):
    indptr, indices, hub = transpose_graph(n)
    reg = cs.transpose_regime(indptr, with_self, sms)
    print("%d SMs, N + 1 = %d (end_bit %d), capacity %d: %d eff_fill passes, %d slot_rows passes" % (
        sms, reg["rows"], reg["end_bit"], reg["cap"], reg["fill_passes"], reg["slot_passes"]))
    assert reg["fill_passes"] >= 3 and reg["slot_passes"] >= 3
    wp, wi, ws = cs.transpose_ref(indptr, indices, with_self)
    E, cap, nnz = int(wp[-1]), reg["cap"], len(indices)
    d_ptr, d_idx = dev(indptr), dev(indices)
    runs = {s: [transpose(gs, d_ptr, d_idx, n, nnz, with_self, s) for _ in range(2)] for s in (False, True)}
    for s, (a, b) in runs.items():
        for x, y, what in zip(a, b, ("t_indptr", "t_indices", "t_slot")):
            if x is not None:
                same(x, y, "slots=%s: %s of two calls" % (s, what))
    tp, ti, ts = runs[True][0]
    body = slice(LEAD, LEAD + cap)
    same(tp, np.concatenate([np.full(LEAD, S64), wp, np.full(TRAIL, S64)]).astype(np.int64), "t_indptr")
    same(ti[LEAD:LEAD + E], wi.astype(np.int32), "t_indices[:E]")
    same(ts[LEAD:LEAD + E], ws.astype(np.int32), "t_slot[:E]")
    for t, what in ((ti, "t_indices"), (ts, "t_slot"), (runs[False][0][1], "plain t_indices")):
        assert (t[:LEAD] == S32).all() and (t[LEAD + cap:] == S32).all(), what + ": a margin was written"
        assert not (t[body] == S32).any(), what + ": a slot was never written"
    same(runs[False][0][0], tp, "plain t_indptr against the slots call")
    same(runs[False][0][1], ti, "plain t_indices against the slots call, tail included")
    got = gs.ops.csr_transpose(d_ptr, d_idx, with_self=with_self, slots=True)
    for g, w, what in zip(got, (tp, ti, ts), ("t_indptr", "t_indices", "t_slot")):
        same(g, w[LEAD:LEAD + len(g)], "ops.csr_transpose " + what)
    assert wp[n + 1] - wp[n] > cs.TRANSPOSE_HUB // 100                  # the dummy row N is an in-degree hub too


# ---------------------------------------------------------------- gs_dropout_apply
@pytest.mark.parametrize("mode", cs.DROPOUT_MODES)
@pytest.mark.parametrize("F", cs.DROPOUT_FS)
def test_dropout_apply_on_every_regime(gs, sms, F, mode):
    reg = cs.dropout_regime(F, sms)
    print("%d SMs, F %d, %s: %d rows, %d quads, %d passes, stride %% quads per row = %d" % (
        sms, F, mode, reg["rows"], reg["quads"], reg["passes"], reg["stride_mod_quads"]))
    assert reg["passes"] >= 3
    rows, group = reg["rows"], cs.DROPOUT_GROUP[mode]
    rs = np.random.RandomState(F * 7 + len(mode))
    site = (2**40 + 17, 2**32 + 9, 0.37)
    scale = 0.3 if group > 1 else 1.0
    x_rows = -(-rows // group)
    x0 = np.full((LEAD + x_rows + TRAIL, F + 3), np.nan, np.float32)
    x0[:, 1:1 + F] = rs.randn(len(x0), F)
    o0 = rs.randn(LEAD + rows + TRAIL, F + 3).astype(np.float32) if mode == "group" else \
        np.full((LEAD + rows + TRAIL, F + 3), np.nan, np.float32)
    pos = None
    if mode == "pos_ids":
        pos = rs.randint(2**30, 2**31 - 1, size=rows).astype(np.int32)
        pos[:3] = [0, 2**31 - 1, 2**30]
    region = (slice(LEAD, LEAD + rows), slice(1, 1 + F))
    x_in = x0[LEAD:LEAD + x_rows, 1:1 + F]
    want = cs.dropout_ref(x_in, site, rows, group, scale, pos, acc=o0[region] if mode == "group" else None)
    got = []
    for _ in range(2):
        xb = dev(x0)
        x = xb[LEAD:LEAD + x_rows, 1:1 + F]
        ob = xb if mode == "in_place" else dev(o0)
        out = ob[region]
        gs.ops.dropout_apply(x, site, rows=rows, group=group, scale=scale, out=out, accumulate=mode == "group",
                             pos_ids=None if pos is None else dev(pos))
        got.append(ob.cpu().numpy())
    same(got[0], got[1], "two calls")
    same_frame(got[0], x0 if mode == "in_place" else o0, region, want, "out")


# ---------------------------------------------------------------- gs_quantize_rows_i8 and Int8Features
def quant_input(rs, n, F):
    x = (rs.randn(n, F) * 10.0 ** rs.uniform(-4, 4, size=(n, 1))).astype(np.float32)
    k = np.arange(n)
    x[k % 997 == 5] = 0                                              # all-zero rows: s = 0
    x[k % 991 == 7] = np.float32(1e-44)                              # a / 127 rounds to zero: every q = 0
    tie = k % 983 == 11                                              # s = 1, x on half-integers: round half to even
    x[tie] = (np.arange(F) % 9 - 4 + 0.5).astype(np.float32)
    x[tie, 0] = 127.0
    return x


@pytest.mark.parametrize("F", cs.QUANT_FS)
def test_quantize_rows_i8_on_every_regime(gs, sms, F):
    n = cs.quant_rows(sms)
    p = cs.passes("quantize_rows_i8_kernel", n, sms)
    print("%d SMs, F %d: %d rows, %d warp passes" % (sms, F, n, p))
    assert p >= 3
    x = quant_input(np.random.RandomState(F), n, F)
    pitch = int8_rows.pitch(F)
    assert pitch == gs._lib.lib().gs_i8row_pitch(F)
    xs = np.full((n, F + 3), np.nan, np.float32)                   # ldx > F: columns past F are never read
    xs[:, :F] = x
    want = int8_rows.quantize_rows(x)
    got = []
    for _ in range(2):
        buf, view = framed((n, pitch), S8, torch.uint8)
        gs.ops.quantize_rows_i8(dev(xs)[:, :F], out=view)
        got.append(buf.cpu().numpy())
    same(got[0], got[1], "two calls")
    same_frame(got[0], np.full(got[0].shape, S8, np.uint8), slice(LEAD, LEAD + n), want, "int8 rows")


def test_int8_features_quantised_in_chunks(gs, sms, monkeypatch):
    from graphsage_b200 import int8_features
    F = 37
    n = cs.quant_rows(sms)
    x = quant_input(np.random.RandomState(3), n, F)
    x[-1] = 0                                                        # the dummy row
    whole = gs.ops.quantize_rows_i8(dev(x)).cpu()
    chunk = n // 3 + 11                                              # three chunks, the last one partial
    monkeypatch.setattr(int8_features, "QUANTIZE_CHUNK_BYTES", 4 * F * chunk)
    t = gs.Int8Features(x)
    assert not t.rows.is_cuda and -(-n // chunk) == 3
    same(t.rows, whole, "Int8Features of a host table in chunks against one launch")
    same(whole, int8_rows.quantize_rows(x), "one launch against the oracle")


# ---------------------------------------------------------------- gs_cast_rows_bf16
@pytest.mark.parametrize("kind", ["vector", "scalar"])
def test_cast_rows_bf16_on_every_regime(gs, sms, kind):
    vec = kind == "vector"
    F, pitch = cs.CAST_VEC if vec else cs.CAST_SCALAR
    n = cs.cast_rows(pitch, vec, sms)
    kernel = "cast_rows_bf16_kernel" if vec else "cast_rows_bf16_scalar_kernel"
    p = cs.passes(kernel, n * (pitch // 8 if vec else pitch), sms)
    print("%d SMs, %s: F %d, out_pitch %d, %d rows, %d passes" % (sms, kernel, F, pitch, n, p))
    assert p >= 3
    rs = np.random.RandomState(pitch)
    ldx = pitch if vec else F + 3
    x = np.full((n, ldx), np.nan, np.float32)                        # columns past F are never read
    x[:, :F] = rs.randint(0, 2**32, size=(n, F), dtype=np.uint64).astype(np.uint32).view(np.float32)
    sv = cs.bf16_special_values()
    at = rs.choice(n * F, size=40 * len(sv), replace=False)
    xf = x[:, :F].copy()
    xf.reshape(-1)[at] = np.resize(sv, len(at))
    x[:, :F] = xf
    assert set(cs.bf16_bits(sv).tolist()) <= set(cs.bf16_bits(xf).reshape(-1).tolist())
    want = np.zeros((n, pitch), np.uint16)
    want[:, :F] = cs.bf16_bits(xf)
    init = np.full((LEAD + n + TRAIL, pitch), 0x5A5A, np.uint16)
    xd = dev(x)
    got = []
    for _ in range(2):
        buf = dev(init.view(np.int16)).view(torch.bfloat16)
        view = buf[LEAD:LEAD + n]
        assert (view.data_ptr() % 16 == 0) or not vec
        call(gs, "gs_cast_rows_bf16", ptr(xd), n, F, ldx, ptr(view), pitch)
        got.append(bits(buf))
    same(got[0], got[1], "two calls")
    same_frame(got[0], init, slice(LEAD, LEAD + n), want, "bf16 rows, pad columns zeroed")


# ---------------------------------------------------------------- halo staging over an emulated 3-shard table
def padded_rows(feats, pitch):
    """The rows as every emulated shard buffer holds them: NaN past F."""
    t = np.full((len(feats), pitch), np.nan, np.float32)
    t[:, :feats.shape[1]] = feats
    return t


def halo_stage(gs, emu, lists, capacity):
    """halo begin -> claim per list -> fetch -> translate per list, into framed sentinel outputs: (count, stage_ids
    buffer, staging buffer, locator buffers) on the host."""
    n_glob = cs.HALO_N + 1
    claim = torch.empty((n_glob,), dtype=torch.int32, device="cuda")
    count = torch.empty((1,), dtype=torch.int32, device="cuda")
    sid, sidv = framed((capacity,), -7, torch.int32)
    stg, stgv = framed((capacity, emu.pitch), -12345.0, torch.float32)
    call(gs, "gs_halo_begin", ptr(claim), n_glob, ptr(count))
    for t in lists:
        call(gs, "gs_halo_claim", emu.c_table(), ptr(t), t.numel(), ptr(claim), ptr(count), ptr(sidv), capacity)
    call(gs, "gs_halo_fetch", emu.c_table(), emu.shape[1], emu.pitch, ptr(sidv), ptr(count), capacity, ptr(stgv),
         emu.pitch)
    locs = []
    for t in lists:
        lb, lv = framed((t.numel(),), S32, torch.int32)
        call(gs, "gs_halo_translate", emu.c_table(), ptr(t), t.numel(), ptr(claim), ptr(lv))
        locs.append(lb.cpu().numpy())
    return int(count.item()), sid.cpu().numpy(), stg.cpu().numpy(), locs


@pytest.mark.parametrize("F", cs.HALO_FS)
def test_halo_staging_on_every_regime(gs, sms, F):
    remote_n = cs.halo_remote()
    rows_pass = cs.stride("halo_fetch_kernel", 1, sms)
    print("%d SMs, F %d: %d ids, %d claim passes; %d remote rows, %.1f fetch passes of %d rows, %d column steps" % (
        sms, F, cs.HALO_IDS, cs.passes("halo_claim_kernel", cs.HALO_IDS, sms), remote_n, remote_n / rows_pass,
        rows_pass, cs.halo_steps(F)))
    assert remote_n >= 3 * rows_pass and cs.passes("halo_claim_kernel", cs.HALO_IDS, sms) >= 3
    feats = np.random.RandomState(F).randn(cs.HALO_N, F).astype(np.float32)
    emu = EmulatedShards(feats, cs.HALO_SPLIT, cs.HALO_MY)
    try:
        lists_np, late = cs.halo_lists(seed=F)                           # late remote ids: only past 2 claim passes
        rule = [cs.rule_locators(x, cs.HALO_SPLIT, cs.HALO_MY, cs.HALO_N) for x in lists_np]
        every, every_rule = np.concatenate(lists_np), np.concatenate(rule)
        remote = np.unique(every[every_rule < 0])
        assert len(remote) == remote_n and np.isin(late, remote).all()
        capacity = remote_n + 50
        table = padded_rows(feats, emu.pitch)
        p4 = (F + 3) // 4 * 4                                              # a row's float4 units: round_up(F, 4) floats
        lists = [dev(x) for x in lists_np]
        for rep in range(2):
            count, sid, stg, locs = halo_stage(gs, emu, lists, capacity)
            assert count == remote_n, rep
            staged = sid[LEAD:LEAD + count].astype(np.int64)
            assert np.array_equal(np.sort(staged), remote), "every remote id takes exactly one slot"
            assert (sid[:LEAD] == -7).all() and (sid[LEAD + count:] == -7).all()
            init = np.full(stg.shape, -12345.0, np.float32)
            same_frame(stg, init, (slice(LEAD, LEAD + count), slice(0, p4)), table[staged, :p4],
                       "staged rows (run %d)" % rep)
            for x, want, got in zip(lists_np, rule, locs):
                assert (got[:LEAD] == S32).all() and (got[LEAD + len(x):] == S32).all()
                got = got[LEAD:LEAD + len(x)]
                local = want >= 0
                same(got[local], want[local].astype(np.int32), "local locators")
                slot = -got[~local].astype(np.int64) - 1
                assert ((slot >= 0) & (slot < count)).all() and np.array_equal(staged[slot], x[~local])
    finally:
        emu.close()


def test_translate_ids_on_every_regime(gs, sms):
    p = cs.passes("translate_ids_kernel", cs.HALO_IDS, sms)
    print("%d SMs: %d ids, %d passes" % (sms, cs.HALO_IDS, p))
    assert p >= 3
    feats = np.random.RandomState(4).randn(cs.HALO_N, 8).astype(np.float32)
    every = np.arange(cs.HALO_N)
    rep = every[cs.rule_locators(every, cs.HALO_SPLIT, cs.HALO_MY, cs.HALO_N) < 0][::5]
    emu = EmulatedShards(feats, cs.HALO_SPLIT, cs.HALO_MY, replica_ids=rep)
    try:
        ids = cs.halo_ids(seed=5)
        want = cs.rule_locators(ids, cs.HALO_SPLIT, cs.HALO_MY, cs.HALO_N, rep).astype(np.int32)
        assert (want < 0).any() and (want > emu.n_local).any()
        d_ids = dev(ids)
        got = []
        for _ in range(2):
            buf, view = framed((len(ids),), S32, torch.int32)
            call(gs, "gs_translate_ids", emu.c_table(), ptr(d_ids), len(ids), ptr(view))
            got.append(buf.cpu().numpy())
        same(got[0], got[1], "two calls")
        same_frame(got[0], np.full(got[0].shape, S32, np.int32), slice(LEAD, LEAD + len(ids)), want, "locators")
    finally:
        emu.close()


def test_halo_fetch_clips_count_to_capacity(gs, sms):
    F = 1500
    feats = np.random.RandomState(6).randn(cs.HALO_N, F).astype(np.float32)
    emu = EmulatedShards(feats, cs.HALO_SPLIT, cs.HALO_MY)
    try:
        every = np.arange(cs.HALO_N)
        remote = np.random.RandomState(7).permutation(
            every[cs.rule_locators(every, cs.HALO_SPLIT, cs.HALO_MY, cs.HALO_N) < 0]).astype(np.int32)
        capacity = 3 * cs.stride("halo_fetch_kernel", 1, sms) + 5
        assert len(remote) >= capacity + 40
        count = torch.tensor([len(remote)], dtype=torch.int32, device="cuda")
        stage_ids = dev(remote)                                   # ids past capacity are remote rows: none may be read
        buf, view = framed((capacity + 40, emu.pitch), -12345.0, torch.float32)      # 40 rows a fetch must not reach
        call(gs, "gs_halo_fetch", emu.c_table(), F, emu.pitch, ptr(stage_ids), ptr(count), capacity, ptr(view),
             emu.pitch)
        init = np.full(tuple(buf.shape), -12345.0, np.float32)
        p4 = (F + 3) // 4 * 4
        same_frame(buf, init, (slice(LEAD, LEAD + capacity), slice(0, p4)),
                   padded_rows(feats, emu.pitch)[remote[:capacity].astype(np.int64), :p4], "rows up to capacity only")
    finally:
        emu.close()


# ---------------------------------------------------------------- HostFeatures.stage and gs_host_fetch
def host_table(gs, dtype, F, n):
    """(the table HostFeatures takes, [n + 1, pitch] bits of the rows as its working set holds them)."""
    rs = np.random.RandomState(F + n)
    x = rs.randn(n + 1, F).astype(np.float32)
    x[n] = 0
    if dtype == "int8":
        t = gs.Int8Features(x)
        return t, bits(t.rows)
    pitch = gs.ops.pad_cols(F)
    if dtype == "bf16":
        t = torch.from_numpy(x).to(torch.bfloat16)
        full = torch.zeros((n + 1, pitch), dtype=torch.bfloat16)
    else:
        t = torch.from_numpy(x)
        full = torch.zeros((n + 1, pitch), dtype=torch.float32)
    full[:, :F] = t
    return t, bits(full)


def ws_bytes(hf):
    return hf.ws.view(torch.uint8)


@pytest.mark.parametrize("cache", ["none", "fill"])
@pytest.mark.parametrize("dtype,F", cs.HOST_CASES)
def test_host_staging_on_every_regime(gs, sms, dtype, F, cache):
    n, C = cs.host_sizes(dtype, F, sms)
    C = C if cache == "fill" else 0
    rv = cs.host_row_units(dtype, F)
    rs = np.random.RandomState(F + C)
    table, rows = host_table(gs, dtype, F, n)
    cache_ids = np.sort(rs.choice(n, size=C, replace=False)) if C else None
    lists = [rs.permutation(n).astype(np.int32), rs.randint(-3, n + 3, size=n // 4).astype(np.int32),
             np.array([n, -1, cs.INT32_MAX, 0, n - 1, -2**31, n + 1], np.int32)]
    staged_ref, tr_ref = cs.stage_ref(n, lists, np.zeros(0, np.int64) if cache_ids is None else cache_ids)
    count_ref = len(staged_ref)
    fill, stage = cs.host_outer(C * rv, sms), cs.host_outer(count_ref * rv, sms)
    print("%d SMs, %s F %d (%d units a row), %d rows, %d cached: fill %.1f strides / %d outer passes, staging %d rows "
          "%.1f strides / %d outer passes" % (sms, dtype, F, rv, n, C, fill[0], fill[1], count_ref, stage[0], stage[1]))
    assert (C == 0 and stage[1] >= 3) or (fill[1] >= 3 and 1 < stage[0] < 8)
    hf = gs.HostFeatures(table, cache_ids=cache_ids)
    try:
        head = C + 1
        same(hf.ws[:head], np.concatenate([rows[cache_ids if C else np.zeros(0, np.int64)],
                                           np.zeros((1, rows.shape[1]), rows.dtype)]), "cached rows and the zero row")
        S = sum(len(x) for x in lists)
        hf.reserve(S)
        lists_d = [dev(x) for x in lists]
        for rep in range(2):
            ws_bytes(hf)[head:] = S8
            ws, tr = hf.stage(lists_d)
            count = int(hf.count)
            assert count == count_ref
            full = bits(hf.ws)
            assert full.shape == (head + S, rows.shape[1])
            # the working-set row of every id: cache slots and the zero row exactly as the oracle's, staged ids once each
            slot_of, moved = np.full(n, -1, np.int64), []
            for x, got, want in zip(lists, tr, tr_ref):
                got = got.cpu().numpy().astype(np.int64)
                fixed = want < head
                assert np.array_equal(got[fixed], want[fixed])
                moved.append((x[~fixed].astype(np.int64), got[~fixed]))
                slot_of[moved[-1][0]] = moved[-1][1]
                same(full[got], rows[np.where((x < 0) | (x >= n), n, x)], "rows the translated ids address")
            assert all(np.array_equal(slot_of[sx], r) for sx, r in moved), "an id took two slots"
            slots = slot_of[staged_ref]
            assert np.array_equal(np.sort(slots), head + np.arange(count)), "the staged ids fill slots 0 .. count - 1"
            same(full[slots], rows[staged_ref], "staged rows")
            assert (full[head + count:].view(np.uint8) == S8).all(), "a row past the count was written"
            same(full[:head - 1], rows[cache_ids] if C else full[:0], "cached rows after the stage")
            assert not full[head - 1].any()
    finally:
        hf.close()


def test_host_fetch_clips_count_to_capacity(gs, sms):
    dtype, F = cs.HOST_CASES[0]
    n, _ = cs.host_sizes(dtype, F, sms)
    table, rows = host_table(gs, dtype, F, n)
    hf = gs.HostFeatures(table)
    try:
        capacity = n // 2 + 3
        ids = np.random.RandomState(8).permutation(n).astype(np.int32)
        stage_ids = dev(ids)                                       # ids past capacity are valid rows: none may be read
        count = torch.tensor([n], dtype=torch.int32, device="cuda")
        buf, view = framed((capacity + 40, rows.shape[1]), float("nan"), torch.float32)
        gs.ops.host_fetch(hf._alias, hf.row_bytes, stage_ids[:capacity], count, view)
        init = bits(np.full(tuple(buf.shape), np.nan, np.float32))
        same_frame(buf, init, slice(LEAD, LEAD + capacity), rows[ids[:capacity].astype(np.int64)],
                   "rows up to capacity only")
    finally:
        hf.close()


# ---------------------------------------------------------------- R-MAT
RMAT = {}


def rmat_oracle():
    if not RMAT:
        p = cs.RMAT_CSR
        RMAT["csr"] = ormat.rmat_csr(p["scale"], p["n"], p["edge_factor"], *cs.RMAT_ABCD, seed=p["seed"])
    return RMAT["csr"]


def rmat_degrees(gs, p):
    n = p["n"]
    mul, mul_inv, add = ormat.scramble_constants(n)
    buf, view = framed((n,), S32, torch.int32)
    call(gs, "gs_rmat_degrees", p["scale"], n, p["edge_factor"], *cs.RMAT_ABCD, p["seed"], mul, mul_inv, add, ptr(view))
    return buf.cpu().numpy()


def test_rmat_degrees_on_every_regime(gs, sms):
    p = cs.RMAT_DEG
    n = p["n"]
    print("%d SMs: scale %d, n %d, %d passes" % (sms, p["scale"], n, cs.passes("rmat_degrees_kernel", n, sms)))
    assert cs.passes("rmat_degrees_kernel", n, sms) >= 3
    want = cs.rmat_degrees_ref(**p)
    got = [rmat_degrees(gs, p) for _ in range(2)]
    same(got[0], got[1], "two calls")
    same_frame(got[0], np.full(got[0].shape, S32, np.int32), slice(LEAD, LEAD + n), want.astype(np.int32), "degrees")


@pytest.mark.parametrize("long", cs.RMAT_THRESHOLDS)
def test_rmat_csr_on_every_regime(gs, sms, long):
    p = cs.RMAT_CSR
    n = p["n"]
    want_ptr, want_idx = rmat_oracle()
    deg = np.diff(want_ptr)
    thr = cs.rmat_threshold(long, deg)
    long_rows = np.nonzero(deg > thr)[0].astype(np.int64)
    print("%d SMs: scale %d, %d rows (%d fill passes), %d entries, longest row %d; threshold %d: %d long rows" % (
        sms, p["scale"], n, cs.passes("rmat_fill_kernel", n, sms), len(want_idx), deg.max(), thr, len(long_rows)))
    assert cs.passes("rmat_fill_kernel", n, sms) >= 3 and deg.max() > 2 * 64 * 256
    # the degrees first: a fill over a wrong indptr would write outside its buffer
    same(rmat_degrees(gs, p)[LEAD:LEAD + n], deg.astype(np.int32), "degrees")
    mul, mul_inv, add = ormat.scramble_constants(n)
    d_ptr, d_long = dev(want_ptr), dev(long_rows)
    got = []
    for _ in range(2):
        buf, view = framed((len(want_idx),), S32, torch.int32)
        call(gs, "gs_rmat_fill", p["scale"], n, *cs.RMAT_ABCD, p["seed"], mul, mul_inv, add, ptr(d_ptr), ptr(view),
             ptr(d_long) if len(long_rows) else 0, len(long_rows), thr)
        got.append(buf.cpu().numpy())
    same(got[0], got[1], "two calls")
    same_frame(got[0], np.full(got[0].shape, S32, np.int32), slice(LEAD, LEAD + len(want_idx)), want_idx, "indices")
    from graphsage_b200.synthetic import rmat_csr_device
    ip, ix = rmat_csr_device(p["scale"], n, p["edge_factor"], *cs.RMAT_ABCD, seed=p["seed"], long_threshold=thr)
    same(ip, want_ptr, "rmat_csr_device indptr")
    same(ix, want_idx, "rmat_csr_device indices")
