"""GPU: the neighbour samplers where the rest of the suite never reaches them - grid-stride loops that take three or
more passes, max_deg up to 1024, four hops with fanout 64, hub rows of 10^5 and 10^6 entries, rows of degree exactly
k - 1, k, k + 1 and 2k, out-of-range ids, 64-bit counters whose sum carries across 2^32, sampled-block calls past 2^32
and a padded table of more than 2^31 entries.  Every output is compared bit for bit with the oracle: gs_sample_padded,
gs_sample_padded_khop (successive oracle.sample_padded calls at counter + t), gs_sample_csr, gs_build_padded_adj (its
degree vector too), gs_csr_sample_rows, ops.csr_blocks(..., fanouts=) and gs_sample_unigram.

The cases and the Python mirror of the launch grids are in test_sampler_regimes_cpu.py, which checks that the mirror's
constants are the sources' and that every case reaches its regimes on 114 and 132 SMs; here each case asserts its
regimes again for this GPU's SM count and prints them.  Where the C API takes the output buffer it is called directly,
with the buffer pre-filled with a sentinel, so an element that no thread writes fails deterministically."""
import ctypes

import numpy as np
import pytest
import torch

import oracle
import test_sampler_regimes_cpu as cs
from oracle import sampled_blocks as sb

pytestmark = pytest.mark.gpu

SEED = 2**63 + 123
CARRIES = ((2**32 - 1, 1), (2**33 - 3, 5))          # (counter, *counter_dev): the 64-bit sum carries across 2^32


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


def filled(shape, dtype=torch.int32):
    return torch.full(shape, cs.SENTINEL, dtype=dtype, device="cuda")


def word(v):
    """A device counter word (uint64 read as int64: every value here is below 2^63)."""
    return None if v is None else torch.tensor([v], dtype=torch.int64, device="cuda")


def same(got, want, what):
    """got (CUDA tensor) equals want (numpy) bit for bit; on a mismatch name the first elements that differ."""
    g = got.cpu().numpy()
    want = np.asarray(want)
    assert g.shape == want.shape, (what, g.shape, want.shape)
    bad = np.nonzero((g != want).reshape(-1))[0]
    if len(bad):
        pytest.fail("%s: %d of %d elements differ (%d never written); first at %s: got %s, want %s" % (
            what, len(bad), g.size, int((g == cs.SENTINEL).sum()), bad[:5].tolist(), g.reshape(-1)[bad[:5]].tolist(),
            want.reshape(-1)[bad[:5]].tolist()))


def ptr(t):
    return 0 if t is None else t.data_ptr()


# ---------------------------------------------------------------- gs_sample_padded
@pytest.mark.parametrize("md,k", cs.PADDED_CASES)
def test_sample_padded_on_every_regime(gs, sms, md, k):
    c = cs.padded_case(sms, md, k, seed=md + k)
    assert c["passes"] >= 3
    print("%d SMs, max_deg %d, k %d: %d ids x %d = %d elements, %d passes" % (sms, md, k, c["n"], k, c["n"] * k,
                                                                               c["passes"]))
    adj, ids = dev(c["adj"]), dev(c["ids"])
    for counter, cdev in CARRIES:
        assert (counter & 0xFFFFFFFF) + cdev >= 2**32
        out = filled((c["n"], k))
        gs.ops.sample_padded(adj, ids, k, SEED, counter, counter_dev=word(cdev), out=out)
        same(out, oracle.sample_padded(c["adj"], c["ids"], k, SEED, counter + cdev), "counter %d + %d" % (counter, cdev))
    perm = np.random.RandomState(k).permutation(md)[:k].astype(np.int32)
    out = filled((c["n"], k))
    gs.ops.sample_padded(adj, ids, k, 0, 0, col_perm=dev(perm), out=out)
    same(out, oracle.sample_padded(c["adj"], c["ids"], k, 0, 0, col_perm=perm), "col_perm")


# ---------------------------------------------------------------- gs_sample_padded_khop
def khop(gs, adj, seeds, fanouts, counter, cdev):
    lib = gs._lib.lib()
    outs, cnt = [], seeds.numel()
    for k in fanouts:
        cnt *= k
        outs.append(filled((cnt,)))
    H = len(fanouts)
    fan = (ctypes.c_int32 * H)(*fanouts)
    optr = (ctypes.c_void_p * H)(*[ptr(o) for o in outs])
    cd = word(cdev)
    gs._lib.check(lib.gs_sample_padded_khop(ptr(adj), adj.shape[0], adj.shape[1], ptr(seeds), seeds.numel(), fan, H,
                                            SEED, counter, ptr(cd), optr, gs._lib.stream_ptr()))
    return outs


@pytest.mark.parametrize("name,md,fanouts", cs.KHOP_CASES)
def test_khop_on_every_regime(gs, sms, name, md, fanouts):
    c = cs.khop_case(sms, name, md, fanouts, seed=md + len(fanouts))
    print("%d SMs, %s, max_deg %d: %s" % (sms, name, md, cs.require_khop(name, c["regime"])))
    assert ((c["adj"] < 0) | (c["adj"] >= len(c["adj"]))).any()           # the table holds ids the next hop clamps
    adj, seeds = dev(c["adj"]), dev(c["seeds"])
    # hop 0 at counter 2^32 - 1, hop 1 at 2^32; then a plain counter without a device word
    for counter, cdev in ((2**32 - 4, 3), (2**40 + 9, None)):
        outs = khop(gs, adj, seeds, fanouts, counter, cdev)
        cur, ctr = c["seeds"], counter + (cdev or 0)
        for t, (k, o) in enumerate(zip(fanouts, outs)):
            cur = oracle.sample_padded(c["adj"], cur, k, SEED, ctr + t).reshape(-1)
            same(o, cur, "hop %d (counter %d)" % (t + 1, ctr + t))


# ---------------------------------------------------------------- gs_sample_csr
CSR = {}


def csr_graph():
    if not CSR:
        CSR["g"] = cs.csr_graph()
    return CSR["g"]


@pytest.mark.parametrize("k", cs.CSR_KS)
def test_sample_csr_on_every_regime(gs, sms, k):
    indptr, indices, hubs = csr_graph()
    n_nodes = len(indptr) - 1
    ids = cs.csr_ids(sms, n_nodes, hubs, seed=k)
    print("%d SMs, k %d: %s" % (sms, k, cs.require_csr(ids, indptr, k, sms)))
    d_ptr, d_idx, d_ids = dev(indptr), dev(indices), dev(ids)
    lib = gs._lib.lib()
    for rep, pad, (counter, cdev) in ((True, -1, CARRIES[0]), (False, n_nodes, CARRIES[1]), (True, n_nodes, (9, None)),
                                      (False, -1, (2**32, None))):
        out, cd = filled((len(ids), k)), word(cdev)
        gs._lib.check(lib.gs_sample_csr(ptr(d_ptr), ptr(d_idx), n_nodes, ptr(d_ids), len(ids), k, int(rep), SEED, counter,
                                        ptr(cd), pad, ptr(out), gs._lib.stream_ptr()))
        same(out, oracle.sample_csr(indptr, indices, ids, k, SEED, counter + (cdev or 0), rep, pad_id=pad),
             "replace_if_short %s, pad_id %d, counter %d + %s" % (rep, pad, counter, cdev))


# ---------------------------------------------------------------- gs_build_padded_adj
@pytest.mark.parametrize("md", cs.BUILD_MDS)
def test_build_padded_adj_on_every_regime(gs, sms, md):
    c = cs.build_case(sms, md, seed=md)
    print("%d SMs, max_deg %d: %s" % (sms, md, cs.require_build(c, sms)))
    n, counter = c["n"], 2**32 + 3
    adj = filled((n + 1, md))
    deg = torch.full((n,), float("nan"), device="cuda")
    indptr, indices, skip = dev(c["indptr"]), dev(c["indices"]), dev(c["skip"].astype(np.uint8))
    gs._lib.check(gs._lib.lib().gs_build_padded_adj(ptr(indptr), ptr(indices), n, md, ptr(skip), SEED, counter, ptr(adj),
                                                    ptr(deg), gs._lib.stream_ptr()))
    want_adj, want_deg = cs.build_padded_adj_ref(c["indptr"], c["indices"], md, SEED, counter, skip=c["skip"])
    same(adj, want_adj, "adj")
    same(deg.view(torch.int32), want_deg.view(np.int32), "deg")


# ---------------------------------------------------------------- gs_csr_sample_rows and the sampled blocks
def sample_rows(gs, indptr, indices, k, call, layer):
    """gs_csr_sample_rows into sentinel-filled outputs: (indptr, indices) as CUDA tensors."""
    lib = gs._lib.lib()
    n, nnz = len(indptr) - 1, len(indices)
    nbytes = lib.gs_csr_sample_rows_workspace_bytes(n, nnz)
    assert nbytes > 0
    ws = torch.empty((nbytes,), dtype=torch.uint8, device="cuda")
    d_ptr, d_idx = dev(indptr), dev(indices)
    out_ptr = filled((n + 1,), torch.int64)
    args = (ptr(d_ptr), ptr(d_idx), n, nnz, k, SEED, call, layer, ptr(ws), nbytes, ptr(out_ptr))
    gs._lib.check(lib.gs_csr_sample_rows(*args, 0, gs._lib.stream_ptr()))
    out_idx = filled((int(out_ptr[-1]),))
    gs._lib.check(lib.gs_csr_sample_rows(*args, ptr(out_idx), gs._lib.stream_ptr()))
    return out_ptr, out_idx


@pytest.mark.parametrize("k", cs.ROWS_KS)
def test_sample_csr_rows_on_every_regime(gs, sms, k):
    indptr, indices = cs.rows_graph(sms, [k], seed=k)
    print("%d SMs, k %d: %s" % (sms, k, cs.require_rows(indptr, k, sms)))
    for call, layer in ((2**32 + 5, 1), (7, 0)):
        got_ptr, got_idx = sample_rows(gs, indptr, indices, k, call, layer)
        want_ptr, want_idx = sb.sample_rows(indptr, indices, k, SEED, call, layer)
        same(got_ptr, want_ptr, "indptr, call %d" % call)
        same(got_idx, want_idx.astype(np.int32), "indices, call %d" % call)
        if call >= 2**32:               # the call word is truncated to 32 bits: call 2^32 + 5 draws what call 5 draws
            same(got_idx, sb.sample_rows(indptr, indices, k, SEED, call & 0xFFFFFFFF, layer)[1].astype(np.int32),
                 "call %d against call %d" % (call, call & 0xFFFFFFFF))


def sampled_blocks(gs, indptr, indices, seeds, fanouts, call):
    """gs_csr_sampled_blocks_plan / _fill, as ops.csr_blocks calls them, into sentinel-filled outputs."""
    lib, L = gs._lib.lib(), len(fanouts)
    n_nodes, nnz, n = len(indptr) - 1, len(indices), len(seeds)
    d_ptr, d_idx, d_seeds = dev(indptr), dev(indices), dev(seeds)
    fan = (ctypes.c_int32 * L)(*fanouts)
    nbytes = lib.gs_csr_blocks_workspace_bytes(n_nodes, nnz, n, L)
    ws = torch.empty((nbytes,), dtype=torch.uint8, device="cuda")
    counts = filled((2 * L,), torch.int64)
    head = (ptr(d_ptr), ptr(d_idx), n_nodes, nnz, ptr(d_seeds), n, L, fan, SEED, call)
    gs._lib.check(lib.gs_csr_sampled_blocks_plan(*head, ptr(ws), nbytes, ptr(counts), gs._lib.stream_ptr()))
    sizes = [int(x) for x in counts.tolist()]
    out_rows = [sizes[2 * l + 2] for l in range(L - 1)] + [n]
    blocks = [(filled((sizes[2 * l],)), filled((sizes[2 * l],), torch.int64), filled((sizes[2 * l + 1],)),
               filled((out_rows[l],))) for l in range(L)]
    arrs = [(ctypes.c_void_p * L)(*[ptr(b[j]) for b in blocks]) for j in range(4)]
    sz = (ctypes.c_int64 * (2 * L))(*sizes)
    gs._lib.check(lib.gs_csr_sampled_blocks_fill(*head, ptr(ws), nbytes, sz, *arrs, gs._lib.stream_ptr()))
    return blocks


def test_sampled_blocks_on_every_regime(gs, sms):
    indptr, indices = cs.rows_graph(sms, cs.BLOCK_FANOUTS, seed=7)
    seeds = cs.block_seeds(sms, len(indptr) - 1, seed=8)
    call = 2**32 + 5
    want = sb.sampled_blocks(indptr, indices, seeds, cs.BLOCK_FANOUTS, SEED, call)
    print("%d SMs, fanouts %s: %s" % (sms, cs.BLOCK_FANOUTS, cs.require_blocks(want, len(seeds), sms)))
    got = sampled_blocks(gs, indptr, indices, seeds, cs.BLOCK_FANOUTS, call)
    for l, (g, w) in enumerate(zip(got, want)):
        for key, t in zip(("src_ids", "indptr", "indices", "rows"), g):
            same(t, np.asarray(w[key]).astype(t.cpu().numpy().dtype), "block %d %s" % (l, key))
    again = gs.ops.csr_blocks(dev(indptr), dev(indices), dev(seeds), 2, fanouts=cs.BLOCK_FANOUTS, seed=SEED,
                              call=call & 0xFFFFFFFF)
    assert all(torch.equal(a, b) for x, y in zip(got, again) for a, b in zip(x, y))


# ---------------------------------------------------------------- gs_sample_unigram
def test_sample_unigram_zero_weight_runs(gs):
    rs = np.random.RandomState(3)
    mid = rs.randint(0, 4, size=500).astype(np.float64)
    for w in (np.array([0, 0, 0, 3, 0, 1, 5, 0, 0, 0], np.float64), np.array([2.0]),
              np.concatenate([np.zeros(300), mid, np.zeros(700)])):
        cdf = dev(np.cumsum(w ** 0.75))                    # the oracle's own float64 prefix sum
        for counter, cdev in ((2**32 - 1, 1), (11, None)):
            out, cd = filled((20_000,)), word(cdev)
            gs._lib.check(gs._lib.lib().gs_sample_unigram(ptr(cdf), len(w), out.numel(), SEED, counter, ptr(cd), ptr(out),
                                                          gs._lib.stream_ptr()))
            same(out, oracle.sample_unigram(w, out.numel(), SEED, counter + (cdev or 0)), "n %d" % len(w))
            assert (w[out.cpu().numpy()] > 0).all()


# ---------------------------------------------------------------- addresses past 2^31 entries
def test_padded_table_past_2_31_entries(gs):
    nbytes = cs.BIG_ROWS * cs.BIG_MD * 4
    free, _ = torch.cuda.mem_get_info()
    if free < 2 * nbytes:
        pytest.skip("a %.1f GB table needs %.1f GB free on this shared GPU; %.1f GB are" % (nbytes / 1e9, 2 * nbytes / 1e9,
                                                                                          free / 1e9))
    adj = torch.empty((cs.BIG_ROWS, cs.BIG_MD), dtype=torch.int32, device="cuda")
    try:
        cols = torch.arange(cs.BIG_MD, dtype=torch.int64, device="cuda")
        for r0 in range(0, cs.BIG_ROWS, 1 << 16):
            r = torch.arange(r0, min(r0 + (1 << 16), cs.BIG_ROWS), dtype=torch.int64, device="cuda")
            adj[r0:r0 + len(r)] = (cs.BIG_ROWS - 1 - (r[:, None] * 31 + cols[None, :] * 17) % 128).to(torch.int32)
        ids = np.concatenate([np.arange(cs.BIG_ROWS - 300, cs.BIG_ROWS), [0, 5, -1, cs.BIG_ROWS, cs.INT32_MAX,
                                                                           cs.INT32_MIN]]).astype(np.int32)
        assert (ids.astype(np.int64) * cs.BIG_MD >= 2**31).sum() >= 64
        for k in (33, cs.BIG_MD):
            out = filled((len(ids), k))
            gs.ops.sample_padded(adj, dev(ids), k, SEED, 2**32 - 1, counter_dev=word(1), out=out)
            same(out, cs.sample_formula_table(ids, k, SEED, 2**32), "k %d" % k)
        fanouts = [16, 8]
        outs = khop(gs, adj, dev(ids), fanouts, 2**32 - 2, 1)
        cur = ids
        for t, (k, o) in enumerate(zip(fanouts, outs)):
            cur = cs.sample_formula_table(cur, k, SEED, 2**32 - 1 + t).reshape(-1)
            same(o, cur, "hop %d" % (t + 1))
        print("table of %d x %d = %d entries (%.1f GB); ids up to row %d" % (cs.BIG_ROWS, cs.BIG_MD,
                                                                           cs.BIG_ROWS * cs.BIG_MD, nbytes / 1e9,
                                                                           cs.BIG_ROWS - 1))
    finally:
        del adj
        torch.cuda.empty_cache()
