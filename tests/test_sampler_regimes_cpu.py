"""The Python mirror of the neighbour samplers' launch grids (graphsage_b200/csrc/sampler.cu and csr_blocks.cu), the
stress cases that test_zz_gpu_sampler_regimes.py runs on them, and the checks that keep both honest: the mirror's
constants are the sources', every case reaches the regimes it is built for on an H100 PCIe (114 SMs) and an H100 SXM
(132 SMs), the oracle's out-of-range rule for the padded sampler is the header's, and the vectorised references the GPU
file uses equal the oracle.

Every sampler kernel grid-strides over its work with a grid capped at a multiple of the SM count: a thread (or a warp)
only loops when the work exceeds one pass of the capped grid.  So every case computes the passes it reaches from the SM
count, and the sizes are derived from the SM count, so no case falls back under its cap on a GPU with more SMs."""
import math
import os
import re

import numpy as np
import pytest

import oracle
from oracle import sampled_blocks as sb
from oracle.philox import mulhi32
from oracle.sampler import _draws

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "graphsage_b200", "csrc")
SM_COUNTS = (114, 132)   # H100 PCIe, H100 SXM
STREAM_BUILD = 0x10000000
INT32_MIN, INT32_MAX = -2**31, 2**31 - 1
SENTINEL = -777_777      # pre-filled into every output: an element that no thread writes keeps it

# ---------------------------------------------------------------- the mirror of the launch grids
# kernel: (threads or warps per block = the items one block takes per pass, grid cap in blocks per SM)
GRIDS = {
    "sample_padded_kernel": (256, 8),          # one thread per output element
    "sample_padded_khop_kernel": (512, 2),     # one thread per output element of every hop
    "sample_csr_kernel": (8, 8),               # one warp per requested id
    "build_padded_adj_kernel": (8, 4),         # one warp per row, the dummy row N included
    "blk_fill_kernel": (8, 16),                # one warp per block row (gs_csr_sample_rows: per node)
    "blk_mark_kernel": (8, 16),                # one warp per node of the previous level
}


def stride(kernel, items, sms):
    """Items one pass of the capped grid covers: min(ceil(items / per_block), cap * SMs) * per_block."""
    per_block, cap = GRIDS[kernel]
    return max(1, min(-(-items // per_block), cap * sms)) * per_block


def passes(kernel, items, sms, grid_items=None):
    """Passes of the grid-stride loop over `items` (the grid sized for grid_items, which defaults to items)."""
    return -(-items // stride(kernel, items if grid_items is None else grid_items, sms)) if items else 0


def _source(name):
    with open(os.path.join(CSRC, name)) as f:
        return f.read()


def _function(src, name):
    m = re.search(r"^(?:static )?int32_t %s\(.*?^}$" % name, src, re.S | re.M)
    assert m, name
    return m.group(0)


def _sm_caps(body):
    return [int(x) for x in re.findall(r"sm_count\(\)\s*\*\s*(\d+)", body)]


def test_mirror_constants_equal_the_sources():
    src = _source("sampler.cu")
    for fn, kernel, blocks in (("gs_sample_padded", "sample_padded_kernel", "(total + 255) / 256"),
                               ("gs_sample_padded_khop", "sample_padded_khop_kernel", "(total + 511) / 512"),
                               ("gs_sample_csr", "sample_csr_kernel", "(n + 7) / 8"),
                               ("gs_build_padded_adj", "build_padded_adj_kernel", "(n_nodes + 1 + 7) / 8")):
        body = _function(src, fn)
        per_block, cap = GRIDS[kernel]
        assert _sm_caps(body) == [cap], fn
        assert blocks in body, fn
        threads = re.findall(r"%s<<<\(unsigned\)blocks,\s*(\d+)," % kernel, body)
        assert threads == [str(per_block if per_block > 32 else per_block * 32)], fn
    # the warp kernels: 8 warps of a 256-thread block
    assert "warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5" in src
    assert "const int64_t warp = (int64_t)blockIdx.x * 8 + w;" in src and "nwarps = (int64_t)gridDim.x * 8;" in src
    assert "u <= n_nodes" in src                                   # the dummy row N is built by the same loop
    blk = _source("csr_blocks.cu")
    assert re.findall(r"constexpr int kBlkThreads = (\d+);", blk) == ["256"]
    assert "constexpr int kBlkWarps = kBlkThreads / 32;" in blk
    for fn in ("blocks_plan", "blocks_fill"):
        body = _function(blk, fn)
        assert "const int64_t max_warp_blocks = (int64_t)sm_count() * 16;" in body, fn
    assert "mark<<<blk_grid(prev_cap, kBlkWarps, max_warp_blocks)" in _function(blk, "blocks_plan")
    assert "fill<<<blk_grid(n_local - 1, kBlkWarps, max_warp_blocks)" in _function(blk, "blocks_fill")
    rows = _function(blk, "gs_csr_sample_rows")
    assert "blk_grid(n_nodes, gs::kBlkWarps, (int64_t)gs::sm_count() * 16)" in rows
    assert "static unsigned blk_grid(int64_t items, int64_t per_block, int64_t max_blocks)" in blk


def test_stride_mirror():
    assert stride("sample_padded_kernel", 99_456, 132) == 389 * 256
    assert stride("sample_padded_kernel", 10**7, 132) == 270_336
    assert stride("sample_padded_khop_kernel", 133_120, 132) == 260 * 512           # the bench shape: one pass
    assert passes("sample_padded_khop_kernel", 133_120, 114) == 2                  # two on an H100 PCIe
    assert stride("sample_csr_kernel", 10**6, 132) == 8_448
    assert stride("build_padded_adj_kernel", 232_966, 132) == 4_224
    assert passes("build_padded_adj_kernel", 232_966, 132) == 56                   # a Reddit-sized table
    assert stride("blk_fill_kernel", 16_384, 132) == 16_384 and stride("blk_fill_kernel", 10**6, 114) == 14_592
    assert passes("blk_mark_kernel", 100, 132, grid_items=10**6) == 1


# ---------------------------------------------------------------- cases
def _place(rs, deg, values, per, hubs=()):
    """Give `per` random rows each of the degrees in `values`, and one row each of the degrees in `hubs` (all distinct
    rows).  The rows, in that order."""
    at = rs.choice(len(deg), size=per * len(values) + len(hubs), replace=False)
    for i, d in enumerate(values):
        deg[at[i * per:(i + 1) * per]] = d
    deg[at[per * len(values):]] = hubs
    return at


def _csr(rs, deg, n_ids):
    indptr = np.concatenate([[0], np.cumsum(deg)]).astype(np.int64)
    return indptr, rs.randint(0, n_ids, size=int(indptr[-1])).astype(np.int32)


# gs_sample_padded: max_deg x k, n * k over at least three passes; a table whose dummy row is not constant
PADDED_MDS = (1, 33, 128, 1000, 1024)
PADDED_CASES = [(md, k) for md in PADDED_MDS for k in sorted({1, 31, 32, 33, md}) if k <= md]
BAD_IDS = (-1, -5, INT32_MIN, INT32_MAX)       # plus n_rows itself


def padded_table(rs, n_rows, md):
    """int32 [n_rows, md], every row (the dummy row n_rows - 1 too) random ids in [0, n_rows)."""
    return rs.randint(0, n_rows, size=(n_rows, md)).astype(np.int32)


def padded_case(sms, md, k, seed):
    rs = np.random.RandomState(seed)
    n_rows = 3001
    n = -(-int(3.2 * stride("sample_padded_kernel", 10**12, sms)) // k)
    ids = rs.randint(0, n_rows, size=n).astype(np.int64)
    bad = rs.choice(n, size=min(n, 400), replace=False)
    ids[bad] = np.resize(np.array(BAD_IDS + (n_rows,), np.int64), len(bad))
    ids[-5:] = BAD_IDS + (n_rows,)
    return dict(adj=padded_table(rs, n_rows, md), ids=ids.astype(np.int32), n=n,
                passes=passes("sample_padded_kernel", n * k, sms))


# gs_sample_padded_khop: (name, max_deg, fanouts, seeds); the seeds' count as a function of one pass's size
def _khop_seeds(name, s):
    return {"1 hop [64]": -(-int(3.2 * s) // 64),
            "bench [10, 25], 512 seeds": 512,
            "bench [10, 25], padded": -(-int(2.5 * s) // 260),
            "3 hops [64, 64, 2]": -(-int(1.25 * s) // (64 * 65)),
            "4 hops [64, 64, 4, 2]": 64}[name]


KHOP_CASES = [("1 hop [64]", 64, [64]), ("bench [10, 25], 512 seeds", 128, [10, 25]),
              ("bench [10, 25], padded", 128, [10, 25]), ("3 hops [64, 64, 2]", 1000, [64, 64, 2]),
              ("4 hops [64, 64, 4, 2]", 1024, [64, 64, 4, 2])]


def khop_regime(n_seeds, fanouts, sms):
    counts = np.cumprod([n_seeds] + list(fanouts))[1:]
    total = int(counts.sum())
    s = stride("sample_padded_khop_kernel", total, sms)
    bounds = np.cumsum(counts)[:-1]
    return dict(total=total, stride=s, passes=-(-total // s),
                hop_changes=int((bounds > s).sum()))       # boundaries a thread's own loop steps across


def khop_case(sms, name, md, fanouts, seed):
    rs = np.random.RandomState(seed)
    n_rows = 3001
    adj = padded_table(rs, n_rows, md)
    hit = rs.rand(n_rows, md) < 0.03                             # entries the next hop must clamp
    adj[hit] = rs.choice(np.array([-3, INT32_MIN, n_rows, INT32_MAX], np.int32), size=int(hit.sum()))
    n_seeds = _khop_seeds(name, 512 * 2 * sms)
    seeds = rs.randint(0, n_rows, size=n_seeds).astype(np.int32)
    seeds[:3] = [-1, n_rows, INT32_MAX]
    return dict(adj=adj, seeds=seeds, regime=khop_regime(n_seeds, fanouts, sms))


def require_khop(name, reg):
    what = "%d elements, %d passes of %d, %d hop boundaries inside a thread's loop" % (
        reg["total"], reg["passes"], reg["stride"], reg["hop_changes"])
    if name.endswith("512 seeds"):
        return what                                             # the bench shape as it is: one pass on 132 SMs
    assert reg["passes"] >= 2, what
    if name.startswith(("3 hops", "4 hops")):
        assert reg["passes"] >= 3 and reg["hop_changes"] >= 1, what
    return what


# gs_sample_csr: one graph with rows of degree 0, k - 1, k, k + 1, 2k for every k, and hubs of 10^5 and 10^6
CSR_KS = (1, 2, 31, 32)
CSR_HUBS = (100_000, 1_000_000)


def csr_graph(seed=21):
    rs = np.random.RandomState(seed)
    n = 6000
    deg = rs.randint(0, 60, size=n)
    special = sorted({d for k in CSR_KS for d in (0, k - 1, k, k + 1, 2 * k)})
    hubs = _place(rs, deg, special, 25, CSR_HUBS)[-len(CSR_HUBS):]
    indptr, indices = _csr(rs, deg, n)
    return indptr, indices, hubs


def csr_ids(sms, n_nodes, hubs, seed):
    """ids over at least three warp passes; every row many times, the hubs and the special rows included, and -1,
    n_nodes and INT32_MAX."""
    rs = np.random.RandomState(seed)
    n = int(3.2 * stride("sample_csr_kernel", 10**12, sms))
    ids = rs.randint(0, n_nodes, size=n).astype(np.int64)
    ids[rs.choice(n, size=60, replace=False)] = np.resize(hubs, 60)
    ids[rs.choice(n, size=60, replace=False)] = np.resize([-1, n_nodes, INT32_MAX], 60)
    return ids.astype(np.int32)


def require_csr(ids, indptr, k, sms):
    deg = np.diff(indptr)
    valid = (ids >= 0) & (ids < len(deg))
    d = set(deg[ids[valid]].tolist())
    missing = {0, k - 1, k, k + 1, 2 * k, *CSR_HUBS} - d
    assert not missing, "degrees %s never requested" % sorted(missing)
    assert (~valid).sum() >= 3
    p = passes("sample_csr_kernel", len(ids), sms)
    assert p >= 3, p
    return "%d ids, %d warp passes" % (len(ids), p)


# gs_build_padded_adj: rows of degree 0, 1, md - 1, md, md + 1, 2 md and hubs of >= 10^5; three or more warp passes
BUILD_MDS = (1, 31, 32, 33, 128, 1024)
BUILD_HUBS = (100_000, 100_003, 131_071)


def build_case(sms, md, seed):
    rs = np.random.RandomState(seed)
    n = int(3.2 * stride("build_padded_adj_kernel", 10**12, sms))
    deg = np.where(rs.rand(n) < 0.5, 0, rs.randint(1, min(2 * md, 40) + 1, size=n))
    special = sorted({0, 1, md - 1, md, md + 1, 2 * md})
    at = _place(rs, deg, special, 24, BUILD_HUBS)
    skip = rs.rand(n) < 0.1
    skip[at[::2]] = False                                        # every degree occurs in rows that are built
    skip[at[-len(BUILD_HUBS):]] = False
    indptr, indices = _csr(rs, deg, n)
    return dict(indptr=indptr, indices=indices, skip=skip, n=n, degrees=special + list(BUILD_HUBS))


def require_build(c, sms):
    n = c["n"]
    s = stride("build_padded_adj_kernel", n + 1, sms)
    p, dummy_pass = -(-(n + 1) // s), n // s
    deg = np.diff(c["indptr"])[~c["skip"]]
    missing = set(c["degrees"]) - set(deg.tolist())
    assert not missing, "degrees %s never built" % sorted(missing)
    assert c["skip"].any()
    assert p >= 3 and dummy_pass >= 1, (p, dummy_pass)
    return "%d rows + the dummy, %d warp passes (the dummy row N in pass %d)" % (n, p, dummy_pass + 1)


def build_padded_adj_ref(indptr, indices, md, seed, counter, skip=None):
    """Vectorised oracle.build_padded_adj: (adj int32 [N + 1, md], deg float32 [N])."""
    indptr = np.asarray(indptr, np.int64)
    indices = np.asarray(indices)
    n = len(indptr) - 1
    lo = indptr[:-1]
    deg = indptr[1:] - lo
    if skip is not None:
        deg = np.where(np.asarray(skip, bool), 0, deg)
    adj = np.full((n + 1, md), n, dtype=np.int32)
    full = np.nonzero(deg == md)[0]
    adj[full] = indices[lo[full, None] + np.arange(md)]
    for rows in np.array_split(np.nonzero((deg > 0) & (deg < md))[0], 8):
        if len(rows):
            r = _draws(seed, counter, md, c2=rows.astype(np.uint32), tag=STREAM_BUILD)
            adj[rows] = indices[lo[rows, None] + mulhi32(r, deg[rows, None].astype(np.uint32)).astype(np.int64)]
    hub = np.nonzero(deg > md)[0]
    if len(hub):
        r = _draws(seed, counter, md, c2=hub.astype(np.uint32), tag=STREAM_BUILD)
        adj[hub] = indices[lo[hub, None] + sb.floyd_positions(r, deg[hub])]
    return adj, deg.astype(np.float32)


# gs_csr_sample_rows / csr_blocks(..., fanouts): rows of degree k - 1, k, k + 1, 2k and a hub, over 3+ fill passes
ROWS_KS = (31, 32, 33, 63, 64, 65, 100, 255, 256)
ROWS_HUB = 100_000
BLOCK_FANOUTS = [100, 33]


def rows_graph(sms, ks, seed):
    """A graph of more than 3 fill passes of nodes: rows of degree k - 1, k, k + 1, 2k for each k in ks, a hub, and
    degrees below 24 elsewhere.  (indptr, indices)."""
    rs = np.random.RandomState(seed)
    n = int(3.3 * stride("blk_fill_kernel", 10**12, sms))
    deg = rs.randint(0, 24, size=n)
    _place(rs, deg, sorted({d for k in ks for d in (k - 1, k, k + 1, 2 * k)}), 30, [ROWS_HUB])
    return _csr(rs, deg, n)


def require_rows(indptr, k, sms):
    n = len(indptr) - 1
    d = set(np.diff(indptr).tolist())
    missing = {k - 1, k, k + 1, 2 * k, ROWS_HUB} - d
    assert not missing, "degrees %s missing" % sorted(missing)
    p = passes("blk_fill_kernel", n, sms)
    assert p >= 3, p
    return "%d nodes, %d fill passes" % (n, p)


def block_seeds(sms, n_nodes, seed):
    rs = np.random.RandomState(seed)
    seeds = rs.randint(0, n_nodes, size=int(3.2 * stride("blk_mark_kernel", 10**12, sms))).astype(np.int32)
    seeds[:3] = [-1, n_nodes, INT32_MAX]
    return seeds


def require_blocks(blocks, n_seeds, sms):
    """The mark passes of every level and the fill passes of every block, from the blocks' sizes."""
    sizes = [len(b["src_ids"]) for b in blocks]            # |V_0|, |V_1|
    mark = [passes("blk_mark_kernel", n_seeds, sms)] + [passes("blk_mark_kernel", m, sms, grid_items=sizes[0] + 10**9)
                                                        for m in sizes[1:]]
    fill = [passes("blk_fill_kernel", m - 1, sms) for m in sizes]
    what = "seeds %d, |V| %s: mark passes %s (seeds, then V_1), fill passes %s" % (n_seeds, sizes, mark, fill)
    assert min(mark) >= 2 and min(fill) >= 2 and mark[0] >= 3, what
    return what


# gs_sample_padded / khop on a table of more than 2^31 entries: row r, column c holds table_entry(r, c)
BIG_MD = 1024
BIG_ROWS = 2**21 + 64                                      # 2^31 + 65,536 entries; rows 2^21 .. lie past 2^31


def table_entry(r, c, n_rows=BIG_ROWS):
    """Ids in the top 128 rows: half of them start past entry 2^31."""
    return n_rows - 1 - (np.asarray(r, np.int64) * 31 + np.asarray(c, np.int64) * 17) % 128


def sample_formula_table(ids, k, seed, counter, n_rows=BIG_ROWS, md=BIG_MD):
    """oracle.sample_padded over the table of table_entry, without building it."""
    ids = oracle.sampler.clamp_rows(ids, n_rows)
    pi = oracle.perm_prefix(seed, counter, md, k)
    return table_entry(ids[:, None], pi[None, :], n_rows).astype(np.int32)


# ---------------------------------------------------------------- the cases reach their regimes
@pytest.fixture(params=SM_COUNTS, ids=lambda s: "%d_SMs" % s)
def sms(request):
    return request.param


@pytest.mark.parametrize("md,k", PADDED_CASES)
def test_padded_cases_take_three_passes(sms, md, k):
    c = padded_case(sms, md, k, seed=md + k)
    assert c["passes"] >= 3
    ids = c["ids"].astype(np.int64)
    assert set(BAD_IDS + (3001,)) <= set(ids.tolist())
    assert c["n"] * k < 2**31


@pytest.mark.parametrize("name,md,fanouts", KHOP_CASES)
def test_khop_cases_reach_their_regimes(sms, name, md, fanouts):
    reg = khop_regime(_khop_seeds(name, 512 * 2 * sms), fanouts, sms)
    require_khop(name, reg)
    if name.endswith("512 seeds"):
        assert reg["total"] == 133_120 and reg["passes"] == (1 if sms == 132 else 2)


def test_csr_case_reaches_its_regimes(sms):
    indptr, indices, hubs = csr_graph()
    ids = csr_ids(sms, len(indptr) - 1, hubs, seed=1)
    for k in CSR_KS:
        require_csr(ids, indptr, k, sms)


@pytest.mark.parametrize("md", BUILD_MDS)
def test_build_cases_reach_their_regimes(sms, md):
    require_build(build_case(sms, md, seed=md), sms)


def test_rows_and_block_cases_reach_their_regimes(sms):
    for k in ROWS_KS:
        indptr, _ = rows_graph(sms, [k], seed=k)
        require_rows(indptr, k, sms)
    indptr, indices = rows_graph(sms, BLOCK_FANOUTS, seed=7)
    seeds = block_seeds(sms, len(indptr) - 1, seed=8)
    require_blocks(sb.sampled_blocks(indptr, indices, seeds, BLOCK_FANOUTS, 123, 2**32 + 5), len(seeds), sms)


# ---------------------------------------------------------------- the oracle and the vectorised references
def test_oracle_clamps_out_of_range_ids_to_the_dummy_row():
    adj = np.arange(40, dtype=np.int32).reshape(8, 5)            # every row distinct: row r holds 5r .. 5r + 4
    ids = np.array([0, -1, 7, 8, -5, INT32_MIN, INT32_MAX, 3, 9], np.int32)
    pi = [4, 0, 2]
    got = oracle.sample_padded(adj, ids, 3, 0, 0, col_perm=pi)
    want = np.array([[4, 0, 2], [39, 35, 37], [39, 35, 37], [39, 35, 37], [39, 35, 37], [39, 35, 37], [39, 35, 37],
                     [19, 15, 17], [39, 35, 37]], np.int32)
    assert np.array_equal(got, want)
    assert got.dtype == np.int32
    # hop ids go through the same rule: row 2 holds an out-of-range id, so its second hop reads the dummy row
    adj2 = adj.copy()
    adj2[2] = [-3, 8, INT32_MAX, 6, 1]
    samples, _ = oracle.sample_khop(adj2, np.array([2], np.int32), [1, 5], 9, 4)   # layer order
    pi1 = oracle.perm_prefix(9, 5, 5, 1)
    hop1 = adj2[2, oracle.perm_prefix(9, 4, 5, 5)]
    want2 = np.array([adj2[h if 0 <= h < 8 else 7, pi1[0]] for h in hop1], np.int32)
    assert np.array_equal(samples[1], hop1) and np.array_equal(samples[2], want2)


@pytest.mark.parametrize("md", [1, 3, 8, 33])
def test_vectorised_build_equals_the_oracle(md):
    rs = np.random.RandomState(md)
    n = 300
    deg = rs.randint(0, 3 * md + 2, size=n)
    _place(rs, deg, sorted({0, 1, md - 1, md, md + 1, 2 * md}) + [200], 4)
    indptr, indices = _csr(rs, deg, n)
    indices[rs.rand(len(indices)) < 0.02] = -2                    # entries are copied as stored
    skip = rs.rand(n) < 0.2
    for sk in (None, skip):
        for seed, counter in ((123, 0), (2**63 + 5, 2**32 + 7)):
            want = oracle.build_padded_adj(indptr, indices, md, seed, counter, skip=sk)
            got = build_padded_adj_ref(indptr, indices, md, seed, counter, skip=sk)
            assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])


def test_formula_table_equals_the_oracle_on_a_small_table():
    n_rows, md = 300, 64
    adj = table_entry(np.arange(n_rows)[:, None], np.arange(md)[None, :], n_rows).astype(np.int32)
    ids = np.array([0, 5, 299, 300, -1, INT32_MAX, INT32_MIN, 170], np.int32)
    for k in (1, 33, 64):
        assert np.array_equal(sample_formula_table(ids, k, 7, 2**32 + 1, n_rows, md),
                              oracle.sample_padded(adj, ids, k, 7, 2**32 + 1))
    assert table_entry(0, 0) == BIG_ROWS - 1 and table_entry(BIG_ROWS - 1, BIG_MD - 1).min() >= BIG_ROWS - 128
    assert (BIG_ROWS - 64) * BIG_MD == 2**31 and BIG_ROWS * BIG_MD >= 2**31 + 1024


def test_sample_calls_mask_to_32_bits_in_the_oracle():
    indptr, indices = _csr(np.random.RandomState(3), np.array([300, 5, 0, 70]), 400)
    for k in (33, 64):
        a = sb.sample_rows(indptr, indices, k, 123, 2**32 + 5, 1)
        b = sb.sample_rows(indptr, indices, k, 123, 5, 1)
        c = sb.sample_rows(indptr, indices, k, 123, 6, 1)
        assert all(np.array_equal(x, y) for x, y in zip(a, b))
        assert not np.array_equal(a[1], c[1])


def test_unigram_oracle_never_draws_a_zero_weight():
    w = np.array([0, 0, 0, 3, 0, 1, 5, 0, 0, 0], np.float64)
    got = oracle.sample_unigram(w, 20_000, 9, 2**32 - 1)
    assert set(np.unique(got).tolist()) == {3, 5, 6}
    assert (oracle.sample_unigram(np.array([2.0]), 100, 1, 0) == 0).all()


def test_floyd_on_a_full_row_is_the_identity():
    """Floyd's algorithm over d = k positions takes position j at step j (every t <= j - 1 is already held), so the
    builder's d == max_deg branch is a fast path of the same table: no output can tell the two apart."""
    rs = np.random.RandomState(0)
    for k in (1, 2, 31, 33, 1024):
        u = rs.randint(0, 2**32, size=(5, k), dtype=np.uint64)
        assert (sb.floyd_positions(u, np.full(5, k)) == np.arange(k)).all()
