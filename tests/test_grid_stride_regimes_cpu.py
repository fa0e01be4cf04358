"""The Python mirror of the launch grids of the CSR transpose, dropout, int8 / bf16 row conversion, staging and R-MAT
kernels (graphsage_b200/csrc/csr_backward.cu, gather.cu, host_table.cu and rmat.cu), the stress cases that
test_zz_gpu_grid_stride_regimes.py runs on them, and the checks that keep both honest: the mirror's constants are the
sources', every case reaches the regimes it is built for on an H100 PCIe (114 SMs) and an H100 SXM (132 SMs), and the
vectorised references the GPU file uses equal the oracle.

Each of these kernels grid-strides over its work with a grid capped at a multiple of the SM count (host_fetch_kernel and
halo_fetch_kernel launch that capped grid whatever the work): a thread or a warp only loops when the work exceeds one
pass.  So the cases are sized from the SM count, and every case computes the passes it reaches."""
import os
import re

import numpy as np
import pytest
import torch

from oracle import dropout as od
from oracle import full_neighbor_dropout as fnd
from oracle import full_neighbor_grad as fng
from oracle import host_stage, int8_rows
from oracle import rmat as ormat
from oracle.philox import philox4x32_10, split64

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "graphsage_b200", "csrc")
SM_COUNTS = (114, 132)   # H100 PCIe, H100 SXM
INT32_MAX = 2**31 - 1

# ---------------------------------------------------------------- the mirror of the launch grids
# kernel: (items one CTA takes per pass, grid cap in CTAs per SM).  Items are threads, or warps where a warp owns an item.
GRIDS = {
    "eff_fill_kernel": (8, 8 * 16),               # one warp per effective row, the dummy row N included
    "slot_rows_kernel": (256, 16),                # one thread per transposed slot (capacity, not entries)
    "dropout_apply_kernel": (256, 16),            # one thread per 4-column quad of a row
    "quantize_rows_i8_kernel": (8, 8),            # one warp per row
    "cast_rows_bf16_kernel": (256, 8),            # one thread per 8-column chunk of out_pitch
    "cast_rows_bf16_scalar_kernel": (256, 8),     # one thread per output element, pad included
    "translate_ids_kernel": (256, 8),             # one thread per id
    "halo_claim_kernel": (256, 8),
    "halo_translate_kernel": (256, 8),            # gs_halo_translate and gs_host_translate
    "halo_fetch_kernel": (8, 2),                  # one warp per staged row; halo_fetch_ctas_per_sm defaults to 2
    "host_fetch_kernel": (256, 3),                # one thread per 16-byte unit, kHostLoads units a grid stride apart
    "rmat_degrees_kernel": (256, 16),             # one thread per row
    "rmat_fill_kernel": (8, 16),                  # one warp per row
}
FIXED_GRID = ("halo_fetch_kernel", "host_fetch_kernel")   # the capped grid is launched whatever the work
HOST_LOADS = 8               # kHostLoads: an outer pass of host_fetch_kernel covers 8 grid strides
HALO_LOADS = 5               # kHaloLoads: a lane's column step is 32 * 5 float4 = 640 columns
LONG_GRID = (64, 256)        # rmat_fill_long_kernel: 64 CTAs of 256 threads per long row


def stride(kernel, items, sms):
    """Items one pass of the grid covers: min(ceil(items / per_cta), cap * SMs) * per_cta (the cap for a fixed grid)."""
    per, cap = GRIDS[kernel]
    ctas = cap * sms if kernel in FIXED_GRID else max(1, min(-(-items // per), cap * sms))
    return ctas * per


def passes(kernel, items, sms):
    return -(-items // stride(kernel, items, sms)) if items else 0


def halo_steps(F):
    """Column steps of a halo_fetch lane: ceil(ceil(F / 4) / (32 * kHaloLoads))."""
    return -(-((F + 3) // 4) // (32 * HALO_LOADS))


def host_outer(units, sms):
    """(grid strides, outer passes) host_fetch_kernel takes over `units` 16-byte units."""
    s = stride("host_fetch_kernel", units, sms)
    return units / s, -(-units // (s * HOST_LOADS))


# ---------------------------------------------------------------- the mirror's constants are the sources'
def _source(name):
    with open(os.path.join(CSRC, name)) as f:
        return f.read()


def _function(src, name):
    m = re.search(r"^(?:static )?int32_t %s\(.*?^}$" % name, src, re.S | re.M)
    assert m, name
    return m.group(0)


def _one(pattern, text, what):
    m = re.findall(pattern, text)
    assert len(m) == 1, (what, m)
    return m[0]


def test_transpose_constants_equal_the_source():
    src = _source("csr_backward.cu")
    threads = int(_one(r"constexpr int kTransposeThreads = (\d+);", src, "kTransposeThreads"))
    body = _function(src, "gs_csr_transpose")
    per, a, b = _one(r"fill_blocks = std::min<int64_t>\(\(P\.rows \+ \d+\) / (\d+), \(int64_t\)gs::sm_count\(\) \* (\d+) \* "
                     r"(\d+)\);", body, "fill_blocks")
    assert (int(per), int(a) * int(b)) == GRIDS["eff_fill_kernel"] and int(per) == threads // 32
    assert "warps = (int64_t)gridDim.x * (kTransposeThreads / 32);" in src and "i <= n_nodes; i += warps" in src
    cap = _one(r"slot_blocks = std::min<int64_t>\(\(P\.cap \+ gs::kTransposeThreads - 1\) / gs::kTransposeThreads, "
               r"\(int64_t\)gs::sm_count\(\) \* (\d+)\);", body, "slot_blocks")
    assert (threads, int(cap)) == GRIDS["slot_rows_kernel"]
    assert "k < cap; k += (int64_t)gridDim.x * blockDim.x" in src
    assert len(re.findall(r"<<<\(unsigned\)(?:fill|slot)_blocks, gs::kTransposeThreads, 0, st>>>", body)) == 3


def _capped(body, kernel, blocks_expr):
    """The CTA cap of a `blocks = blocks_expr; cap = sm_count() * c; blocks = min(...)` launch of a 256-thread kernel."""
    assert blocks_expr in body, (kernel, blocks_expr)
    cap = int(_one(r"int64_t cap = \(int64_t\)gs::sm_count\(\) \* (\d+);", body, kernel))
    assert "if (blocks > cap) blocks = cap;" in body, kernel
    assert re.search(r"%s(?:<\w+>)?<<<\(unsigned\)blocks, 256, 0," % kernel, body), kernel
    return cap


def test_gather_constants_equal_the_source():
    src = _source("gather.cu")
    for fn, kernel, expr, per in (
            ("gs_dropout_apply", "dropout_apply_kernel", "blocks = (total + 255) / 256", 256),
            ("gs_quantize_rows_i8", "quantize_rows_i8_kernel", "blocks = (n + 7) / 8", 8),
            ("gs_cast_rows_bf16", "cast_rows_bf16_kernel", "blocks = ((vec ? n * (out_pitch / 8) : n * out_pitch) + 255) / 256",
             256),
            ("gs_cast_rows_bf16", "cast_rows_bf16_scalar_kernel", "blocks = ((vec ? n * (out_pitch / 8)", 256),
            ("gs_translate_ids", "translate_ids_kernel", "blocks = (n + 255) / 256", 256),
            ("gs_halo_claim", "halo_claim_kernel", "blocks = (n + 255) / 256", 256),
            ("gs_halo_translate", "halo_translate_kernel", "blocks = (n + 255) / 256", 256),
            ("gs_host_translate", "halo_translate_kernel", "blocks = (n + 255) / 256", 256)):
        assert (per, _capped(_function(src, fn), kernel, expr)) == GRIDS[kernel], fn
    assert "const int64_t total = rows * ((F + 3) / 4);" in _function(src, "gs_dropout_apply")
    assert "const bool vec = out_pitch % 8 == 0 && gs::aligned16(out_bf16) && ldx >= ((F + 7) / 8) * 8;" in src
    # every loop above: a thread (or warp) index plus multiples of the whole grid
    grid_loops = re.findall(r"q < total; q \+= \(int64_t\)gridDim\.x \* blockDim\.x\)", src)
    assert len(grid_loops) == 3                                   # dropout, both bf16 casts
    assert len(re.findall(r"i < n; i \+= \(int64_t\)gridDim\.x \* blockDim\.x\)", src)) >= 3
    halo = _function(src, "gs_halo_fetch")
    assert int(_one(r'gs::sm_count\(\) \* gs::tuning\("halo_fetch_ctas_per_sm", (\d+)\)', halo, "halo")) == \
        GRIDS["halo_fetch_kernel"][1]
    assert "halo_fetch_kernel<<<(unsigned)blocks, 256, 0," in halo
    assert int(_one(r"constexpr int kHaloLoads = (\d+);", src, "kHaloLoads")) == HALO_LOADS
    assert "c0 < row_f4; c0 += 32 * kHaloLoads" in src and "if (n > capacity) n = capacity;" in src
    assert "const int chunks = (int)(out_pitch >> 3);" in src


def test_host_table_constants_equal_the_source():
    src = _source("host_table.cu")
    assert int(_one(r"constexpr int kHostLoads = (\d+);", src, "kHostLoads")) == HOST_LOADS
    body = _function(src, "gs_host_fetch")
    assert int(_one(r"const int blocks = gs::sm_count\(\) \* (\d+);", body, "blocks")) == GRIDS["host_fetch_kernel"][1]
    assert "host_fetch_kernel<<<(unsigned)blocks, 256, 0," in body
    assert "u0 < total; u0 += stride * kHostLoads" in src and "const int64_t u = u0 + k * stride;" in src
    assert "if (n > capacity) n = capacity;" in src


def test_rmat_constants_equal_the_source():
    src = _source("rmat.cu")
    deg, fill = _function(src, "gs_rmat_degrees"), _function(src, "gs_rmat_fill")
    for body, kernel, expr in ((deg, "rmat_degrees_kernel", "blocks = (n_nodes + 255) / 256;"),
                               (fill, "rmat_fill_kernel", "blocks = (n_nodes + 7) / 8;")):
        assert expr in body, kernel
        cap = int(_one(r"int64_t cap = \(int64_t\)gs::sm_count\(\) \* (\d+);", body, kernel))
        assert re.search(r"%s<<<\(unsigned\)blocks, 256, 0," % kernel, body), kernel
        assert (GRIDS[kernel][0] * (32 if GRIDS[kernel][0] == 8 else 1), cap) == (256, GRIDS[kernel][1])
    x, t = _one(r"rmat_fill_long_kernel<<<dim3\((\d+), \(unsigned\)n_long\), (\d+),", fill, "long")
    assert (int(x), int(t)) == LONG_GRID
    assert "j < deg; j += (int64_t)gridDim.x * blockDim.x" in src and "y < p.n; y += nwarps" in src
    assert "n_long <= 65535" in fill


def test_stride_mirror():
    assert stride("eff_fill_kernel", 10**9, 114) == 116_736 and stride("eff_fill_kernel", 10**9, 132) == 135_168
    assert stride("slot_rows_kernel", 10**9, 114) == 466_944 and stride("dropout_apply_kernel", 10**9, 132) == 540_672
    assert stride("quantize_rows_i8_kernel", 10**9, 114) == 7_296 and stride("quantize_rows_i8_kernel", 10**9, 132) == 8_448
    assert stride("cast_rows_bf16_kernel", 10**9, 114) == 233_472 and stride("halo_claim_kernel", 10**9, 132) == 270_336
    assert stride("halo_fetch_kernel", 1, 114) == 1_824 and stride("halo_fetch_kernel", 1, 132) == 2_112
    assert stride("host_fetch_kernel", 1, 114) == 87_552 and stride("host_fetch_kernel", 1, 132) == 101_376
    assert stride("rmat_fill_kernel", 10**9, 114) == 14_592 and stride("rmat_degrees_kernel", 10**9, 132) == 540_672
    assert stride("slot_rows_kernel", 1000, 132) == 1024 and passes("slot_rows_kernel", 1000, 132) == 1
    assert halo_steps(640) == 1 and halo_steps(641) == 2 and halo_steps(1281) == 3
    assert host_outer(8 * 101_376 + 1, 132)[1] == 2


# ---------------------------------------------------------------- the cases
# gs_csr_transpose: N + 1 = 2^19 and 2^19 + 1 rows (the two sides of a step of the radix sort's end_bit), rows of 0..6
# entries, empty rows, an out-degree hub of 10^5 entries and entries -1, N, N + 1 and INT32_MAX
TRANSPOSE_NS = (2**19 - 1, 2**19)
TRANSPOSE_HUB = 100_000
TRANSPOSE_BAD = (-1, 0, 1, INT32_MAX)           # added to N where the value is not -1 / INT32_MAX: see transpose_graph


def end_bit(rows):
    """make_transpose_plan's end_bit: the least b >= 1 with 2^b > rows."""
    b = 1
    while (1 << b) <= rows:
        b += 1
    return b


def transpose_graph(n, seed):
    """(indptr int64, indices int32, hub row) of n nodes."""
    rs = np.random.RandomState(seed)
    deg = rs.randint(0, 7, size=n)
    deg[rs.rand(n) < 0.15] = 0
    hub = n // 3
    deg[hub] = TRANSPOSE_HUB
    indptr = np.concatenate([[0], np.cumsum(deg)]).astype(np.int64)
    nnz = int(indptr[-1])
    indices = rs.randint(0, n, size=nnz).astype(np.int64)
    bad = rs.choice(nnz, size=4000, replace=False)
    indices[bad] = np.resize(np.array([-1, n, n + 1, INT32_MAX], np.int64), len(bad))
    return indptr, indices.astype(np.int32), hub


def transpose_regime(indptr, with_self, sms):
    n = len(indptr) - 1
    cap = int(indptr[-1]) + (n + 1) * (1 + int(with_self))
    return dict(rows=n + 1, cap=cap, end_bit=end_bit(n + 1), fill_passes=passes("eff_fill_kernel", n + 1, sms),
                slot_passes=passes("slot_rows_kernel", cap, sms))


# gs_dropout_apply: (F, mode) with rows sized for 3.2 passes of quads; mode: plain (group 1), group (25, a scale,
# accumulate), in place (group 1), pos_ids (group 25, positions above 2^30)
DROPOUT_FS = (1, 5, 602)
DROPOUT_MODES = ("plain", "group", "in_place", "pos_ids")
DROPOUT_GROUP = {"plain": 1, "group": 25, "in_place": 1, "pos_ids": 25}


def dropout_rows(F, sms):
    nc4 = (F + 3) // 4
    return -(-int(3.2 * stride("dropout_apply_kernel", 10**12, sms)) // nc4)


def dropout_regime(F, sms):
    nc4 = (F + 3) // 4
    rows = dropout_rows(F, sms)
    s = stride("dropout_apply_kernel", rows * nc4, sms)
    return dict(rows=rows, quads=rows * nc4, passes=passes("dropout_apply_kernel", rows * nc4, sms),
                stride_mod_quads=s % nc4)


# gs_quantize_rows_i8 and gs_cast_rows_bf16
QUANT_FS = (1, 37, 602, 1536)
CAST_VEC = (602, 608)             # (F, out_pitch): 76 chunks of 8 per row
CAST_SCALAR = (601, 603)          # an odd out_pitch: the scalar kernel


def quant_rows(sms):
    return int(3.2 * stride("quantize_rows_i8_kernel", 10**12, sms))


def cast_rows(out_pitch, vec, sms):
    per_row = out_pitch // 8 if vec else out_pitch
    return -(-int(3.2 * stride("cast_rows_bf16_kernel", 10**12, sms)) // per_row)


# halo staging over an emulated 3-shard table: ids over about 10^6 with repeats, every remote row staged
HALO_N = 15_000
HALO_SPLIT = [0, 5_000, 9_999, HALO_N]
HALO_MY = 1
HALO_IDS = 1_000_000
HALO_FS = (602, 1500, 2000)


def halo_ids(seed):
    rs = np.random.RandomState(seed)
    ids = rs.randint(-3, HALO_N + 3, size=HALO_IDS).astype(np.int64)
    ids[rs.choice(HALO_IDS, size=64, replace=False)] = np.resize([-1, HALO_N, HALO_N + 1, INT32_MAX, -2**31], 64)
    return ids.astype(np.int32)


def halo_lists(seed):
    """The three id lists of the halo staging case (10^6 ids, a copy of the first list's head last).  Half of the remote
    ids first appear 600,000 ids into the second list - in its third claim pass on 114 and 132 SMs - so a claim that
    stops after a pass misses them.  (the lists, those late ids)"""
    rs = np.random.RandomState(seed)
    every = np.arange(HALO_N)
    late = rs.permutation(every[rule_locators(every, HALO_SPLIT, HALO_MY, HALO_N) < 0])[:halo_remote() // 2]
    pool = np.setdiff1d(np.arange(-3, HALO_N + 3), late)
    head = pool[rs.randint(0, len(pool), size=HALO_IDS - 100_000)]
    head[rs.choice(len(head), size=64, replace=False)] = np.resize([-1, HALO_N, HALO_N + 1, INT32_MAX, -2**31], 64)
    tail = rs.randint(-3, HALO_N + 3, size=100_000)
    tail[:len(late)] = late
    ids = np.concatenate([head, rs.permutation(tail)]).astype(np.int32)
    return [ids[:300_000], ids[300_000:], ids[:5000].copy()], late


def halo_remote():
    """Global ids not owned by HALO_MY: the rows the staging fetches (there are no replicas)."""
    return HALO_N - (HALO_SPLIT[HALO_MY + 1] - HALO_SPLIT[HALO_MY])


# HostFeatures.stage: (dtype, F) -> 16-byte units per row; tables sized for 2.3 outer passes of the fetch
HOST_CASES = (("fp32", 37), ("bf16", 602), ("int8", 100))


def host_row_units(dtype, F):
    if dtype == "int8":
        return int8_rows.pitch(F) // 16
    return (F + 7) // 8 * 8 * (4 if dtype == "fp32" else 2) // 16


def host_sizes(dtype, F, sms):
    """(table rows N, cached rows C): the whole table staged takes 2.3 outer passes; a cache of C rows is filled in more
    than 2 outer passes and leaves N - C rows (about 2 strides) to stage."""
    rv = host_row_units(dtype, F)
    outer = HOST_LOADS * stride("host_fetch_kernel", 1, sms)
    return -(-int(2.3 * outer) // rv), -(-int(2.05 * outer) // rv)


# R-MAT
RMAT_CSR = dict(scale=18, n=2**18, edge_factor=20.0, seed=7)         # a row of about 37,000 entries
RMAT_DEG = dict(scale=21, n=2_000_000, edge_factor=2.5, seed=9)      # trimmed: ids >= n fold onto id - n
RMAT_ABCD = (0.57, 0.19, 0.19, 0.05)
RMAT_THRESHOLDS = ("none", "one", 300)


def rmat_threshold(which, deg):
    """long_threshold for rmat_csr_device: past every row, one row long, or a fixed degree."""
    mx = int(deg.max())
    return {"none": mx, "one": mx - 1}.get(which, which)


# ---------------------------------------------------------------- vectorised references
def effective_rows(indptr, indices, with_self=False):
    """oracle.full_neighbor_grad.effective_csr vectorised: (eptr, eidx, src, slot) - each entry's source row and its
    t_slot value (j, -1 for the implicit {N} entry, -2 for the with_self entry)."""
    indptr = np.asarray(indptr, np.int64)
    indices = np.asarray(indices, np.int64)
    n = len(indptr) - 1
    deg = np.diff(indptr)
    cnt = np.concatenate([np.maximum(deg, 1), [1]]) + int(bool(with_self))
    eptr = np.zeros(n + 2, np.int64)
    eptr[1:] = np.cumsum(cnt)
    src = np.repeat(np.arange(n + 1, dtype=np.int64), cnt)
    j = np.arange(int(eptr[-1]), dtype=np.int64) - eptr[src]
    real = j < np.concatenate([deg, [0]])[src]
    eidx = np.full(len(src), n, np.int64)
    v = indices[indptr[src[real]] + j[real]]
    eidx[real] = np.where((v < 0) | (v > n), n, v)
    slot = np.where(real, j, -1)
    if with_self:
        last = j == cnt[src] - 1
        eidx[last] = src[last]
        slot[last] = -2
    return eptr, eidx, src, slot


def transpose_ref(indptr, indices, with_self=False):
    """gs_csr_transpose with t_slot: (t_indptr [N + 2], t_indices [E], t_slot [E]), int64."""
    eptr, eidx, src, slot = effective_rows(indptr, indices, with_self)
    n = len(eptr) - 2
    order = np.argsort(eidx, kind="stable")
    t_indptr = np.zeros(n + 2, np.int64)
    t_indptr[1:] = np.cumsum(np.bincount(eidx, minlength=n + 1))
    return t_indptr, src[order], slot[order]


def dropout_ref(x, site, rows, group=1, scale=1.0, pos=None, acc=None):
    """gs_dropout_apply: out[r] (+)= keep ? (x[r // group] * scale) / keep_prob : 0 at position pos[r] (or r)."""
    seed, call, rate = site
    x = np.asarray(x, np.float32)
    r = np.arange(rows)
    m = od.keep_mask(seed, call, rate, r if pos is None else np.asarray(pos)[:rows], x.shape[1])
    v = np.where(m, (x[r // group] * np.float32(scale)) / od.keep_prob(rate), np.float32(0)).astype(np.float32)
    return v if acc is None else (np.asarray(acc, np.float32) + v).astype(np.float32)


def stage_ref(n_nodes, lists, cache_ids):
    """oracle.host_stage.stage without the table, vectorised: (staged ids in first-sighting order, each list as
    working-set rows)."""
    cache_ids = np.asarray(cache_ids, np.int64).reshape(-1)
    C = len(cache_ids)
    slot = np.full(n_nodes + 1, -1, np.int64)          # working-set row per id; index n_nodes: every invalid id
    slot[cache_ids] = np.arange(C)
    every = np.concatenate([np.asarray(x, np.int64).reshape(-1) for x in lists] + [np.zeros(0, np.int64)])
    clamped = np.where((every < 0) | (every >= n_nodes), n_nodes, every)
    want = every[(clamped < n_nodes) & (slot[clamped] < 0)]
    u, first = np.unique(want, return_index=True)
    staged = u[np.argsort(first, kind="stable")]
    slot[staged] = C + 1 + np.arange(len(staged))
    slot[n_nodes] = C
    out = []
    for x in lists:
        x = np.asarray(x, np.int64).reshape(-1)
        out.append(slot[np.where((x < 0) | (x >= n_nodes), n_nodes, x)])
    return staged, out


def rule_locators(ids, row_start, my, n_nodes, rep=()):
    """The locator rule of gs_translate_ids / gs_halo_translate for locally held ids: remap[id] (own row id - lo, the
    zero row for ids outside [0, N), replica i at n_local + 1 + i); -id - 1 for an id its owner has to supply."""
    ids = np.asarray(ids, np.int64)
    rep = np.asarray(rep, np.int64)
    lo, hi = row_start[my], row_start[my + 1]
    out = -ids - 1
    own = (ids >= lo) & (ids < hi)
    out[own] = ids[own] - lo
    if len(rep):
        pos = np.searchsorted(rep, ids)
        hit = (ids >= 0) & (ids < n_nodes) & (pos < len(rep))
        hit[hit] = rep[pos[hit]] == ids[hit]
        out[hit] = (hi - lo) + 1 + pos[hit]
    out[(ids < 0) | (ids >= n_nodes)] = hi - lo
    return out


def rmat_degrees_ref(scale, n, edge_factor, seed, abcd=RMAT_ABCD):
    """The degree half of oracle.rmat.rmat_csr: int64 [n], without the 128 bytes per edge of the fill."""
    a, b, c, d = abcd
    mul, mul_inv, add = ormat.scramble_constants(n)
    prow = ormat._prow(scale, a, b, c, d)
    y = np.arange(n, dtype=np.int64)
    r = ((y - add) % n) * mul_inv % n
    r2 = r + n
    has2 = r2 < (1 << scale)
    p1 = prow[ormat._popcount(r)]
    p2 = np.where(has2, prow[np.minimum(ormat._popcount(r2), scale)], 0.0)
    lam = (edge_factor * float(n)) * np.where(has2, p1 + p2, p1)
    fl = np.floor(lam)
    ctr = np.zeros((n, 4), dtype=np.uint32)
    ctr[:, 0] = y.astype(np.uint32)
    ctr[:, 3] = ormat.TAG_DEG
    u = (philox4x32_10(ctr, np.array(split64(seed), np.uint32))[:, 0].astype(np.float64) + 0.5) * (1.0 / 4294967296.0)
    return np.minimum(fl + (u < (lam - fl)), 2147483647.0).astype(np.int64)


def bf16_bits(x):
    """f32_to_bf16_rne (gather.cu) restated: NaN keeps its sign and top payload bits with the quiet bit set; every
    other value rounds to nearest even on the upper 16 bits (so FLT_MAX and the values near it round to infinity)."""
    u = np.ascontiguousarray(x, np.float32).view(np.uint32).astype(np.uint64)
    nan = (u & 0x7FFFFFFF) > 0x7F800000
    rne = (u + 0x7FFF + ((u >> 16) & 1)) >> 16
    return np.where(nan, (u >> 16) | 0x40, rne).astype(np.uint16)


def bf16_special_values():
    """float32 values at the edges of the conversion: +-0, subnormals, ties, values rounding up to +-inf, +-inf, NaNs."""
    bits = np.array([0x00000000, 0x80000000, 0x00000001, 0x807FFFFF, 0x00008000, 0x00018000, 0x3F808000, 0x3F818000,
                     0x3F807FFF, 0x7F7FFFFF, 0xFF7FFFFF, 0x7F7F8000, 0x7F7F7FFF, 0x7F800000, 0xFF800000, 0x7FC00000,
                     0xFFC00000, 0x7F800001, 0xFF800001, 0x7FBFFFFF, 0x7F80FFFF, 0x00800000, 0x0080FFFF], np.uint32)
    return bits.view(np.float32)


# ---------------------------------------------------------------- the cases reach their regimes
@pytest.fixture(params=SM_COUNTS, ids=lambda s: "%d_SMs" % s)
def sms(request):
    return request.param


@pytest.mark.parametrize("with_self", [False, True])
@pytest.mark.parametrize("n", TRANSPOSE_NS)
def test_transpose_cases_reach_their_regimes(sms, n, with_self):
    indptr, indices, hub = transpose_graph(n, seed=n % 97)
    reg = transpose_regime(indptr, with_self, sms)
    assert reg["fill_passes"] >= 3 and reg["slot_passes"] >= 3, reg
    assert reg["end_bit"] == 20 and end_bit(2**19 - 1) == 19                 # N + 1 = 2^19 is where end_bit steps
    deg = np.diff(indptr)
    assert deg[hub] == TRANSPOSE_HUB and (deg == 0).sum() > 1000
    assert {-1, n, n + 1, INT32_MAX} <= set(np.unique(indices.astype(np.int64)).tolist())


@pytest.mark.parametrize("F", DROPOUT_FS)
def test_dropout_cases_reach_their_regimes(sms, F):
    reg = dropout_regime(F, sms)
    assert reg["passes"] >= 3, reg
    if F == 602:
        assert reg["stride_mod_quads"] != 0, reg        # a thread's quad moves within the row from pass to pass


def test_conversion_cases_reach_their_regimes(sms):
    for F in QUANT_FS:
        assert passes("quantize_rows_i8_kernel", quant_rows(sms), sms) >= 3
    F, pitch = CAST_VEC
    assert pitch % 8 == 0 and pitch == (F + 7) // 8 * 8
    assert passes("cast_rows_bf16_kernel", cast_rows(pitch, True, sms) * (pitch // 8), sms) >= 3
    F, pitch = CAST_SCALAR
    assert pitch % 2 == 1 and pitch > F
    assert passes("cast_rows_bf16_scalar_kernel", cast_rows(pitch, False, sms) * pitch, sms) >= 3


def test_staging_cases_reach_their_regimes(sms):
    assert passes("halo_claim_kernel", HALO_IDS, sms) >= 3 and passes("translate_ids_kernel", HALO_IDS, sms) >= 3
    assert halo_remote() >= 3 * stride("halo_fetch_kernel", 1, sms)
    assert [halo_steps(F) for F in HALO_FS] == [1, 3, 4]                  # F > 640 and F > 1280
    lists, late = halo_lists(seed=602)
    first = {}
    for i, x in enumerate(lists[1].tolist()):
        first.setdefault(x, i)
    assert min(first[x] for x in late.tolist()) >= 2 * stride("halo_claim_kernel", len(lists[1]), sms)
    assert not np.isin(late, np.concatenate([lists[0], lists[2]])).any() and sum(map(len, lists)) >= HALO_IDS
    total_bytes = 0
    for dtype, F in HOST_CASES:
        rv = host_row_units(dtype, F)
        n, C = host_sizes(dtype, F, sms)
        whole, fill, rest = host_outer(n * rv, sms), host_outer(C * rv, sms), host_outer((n - C) * rv, sms)
        assert whole[1] >= 3 and fill[1] >= 3 and 1 < rest[0] < 8, (dtype, whole, fill, rest)
        assert (n * rv) % stride("host_fetch_kernel", 1, sms) != 0          # a partial last stride
        total_bytes += (n + 1) * rv * 16
    assert host_row_units("int8", 100) == 7 and host_row_units("fp32", 37) == 10
    assert total_bytes < 100e6, total_bytes


def test_rmat_cases_reach_their_regimes(sms):
    deg = rmat_degrees_ref(**RMAT_CSR)
    n = RMAT_CSR["n"]
    assert passes("rmat_fill_kernel", n, sms) >= 3
    assert deg.max() > 2 * LONG_GRID[0] * LONG_GRID[1]                    # a long row takes 3 passes of its grid
    assert (deg > rmat_threshold("one", deg)).sum() == 1
    assert 1000 <= (deg > rmat_threshold(300, deg)).sum() <= 65535
    assert (deg > rmat_threshold("none", deg)).sum() == 0
    assert int(deg.sum()) * 128 < 1.0e9                                   # the oracle's 128 bytes per edge
    assert passes("rmat_degrees_kernel", RMAT_DEG["n"], sms) >= 3 and RMAT_DEG["n"] < 2**RMAT_DEG["scale"]


# ---------------------------------------------------------------- the vectorised references equal the oracle
def _messy_csr(rs, n, degrees):
    deg = np.resize(np.array(degrees), n)
    rs.shuffle(deg)
    indptr = np.concatenate([[0], np.cumsum(deg)]).astype(np.int64)
    indices = rs.randint(-2, n + 3, size=int(indptr[-1])).astype(np.int64)
    indices[rs.rand(len(indices)) < 0.02] = INT32_MAX
    return indptr, indices.astype(np.int32)


@pytest.mark.parametrize("with_self", [False, True])
def test_transpose_ref_equals_the_oracle(with_self):
    rs = np.random.RandomState(5)
    for n, degrees in ((1, [0]), (1, [3]), (40, [0, 1, 2, 33]), (300, [0, 0, 1, 5, 70])):
        indptr, indices = _messy_csr(rs, n, degrees)
        wp, wi, ws = transpose_ref(indptr, indices, with_self)
        op, oi = fng.csr_transpose(indptr, indices, with_self)
        sp, si, ss = fnd.csr_transpose_slots(indptr, indices, with_self)
        assert np.array_equal(wp, op) and np.array_equal(wi, oi)
        assert np.array_equal(wp, sp) and np.array_equal(wi, si) and np.array_equal(ws, ss)
        eptr, eidx, _, _ = effective_rows(indptr, indices, with_self)
        oe = fng.effective_csr(indptr, indices, with_self)
        assert np.array_equal(eptr, oe[0]) and np.array_equal(eidx, oe[1])


def test_dropout_ref_equals_the_oracle():
    rs = np.random.RandomState(6)
    for F in (1, 5, 8, 37):
        x = rs.randn(50, F).astype(np.float32)
        site = (2**40 + 3, 11, 0.35)
        assert np.array_equal(dropout_ref(x, site, 50), od.apply(x, *site))
        pos = rs.randint(2**30, 2**31 - 1, size=50)
        assert np.array_equal(dropout_ref(x, site, 50, pos=pos), od.apply(x, *site, pos=pos))
        # group and scale: row r reads x[r // group], scaled before the division by keep
        want = od.apply(np.repeat(x, 3, axis=0)[:149] * np.float32(0.25), *site)
        assert np.array_equal(dropout_ref(x, site, 149, group=3, scale=0.25), want)
        acc = rs.randn(149, F).astype(np.float32)
        assert np.array_equal(dropout_ref(x, site, 149, group=3, scale=0.25, acc=acc), acc + want)


def test_stage_ref_equals_the_oracle():
    rs = np.random.RandomState(7)
    n = 200
    table = np.vstack([rs.randn(n, 3).astype(np.float32), np.zeros((1, 3), np.float32)])
    lists = [rs.randint(-4, n + 4, size=300), np.zeros(0, np.int64), np.array([n, -1, INT32_MAX, 0, 0, 199])]
    for cache in (np.zeros(0, np.int64), np.array([0, 5, 77, 199]), np.arange(n)):
        ws, tr, staged = host_stage.stage(table, lists, cache)
        got_staged, got_tr = stage_ref(n, lists, cache)
        assert np.array_equal(got_staged, staged)
        assert all(np.array_equal(a, b) for a, b in zip(got_tr, tr))


def test_rule_locators_without_replicas_mark_every_remote_id():
    ids = np.array([-1, 0, 4_999, 5_000, 9_998, 9_999, HALO_N - 1, HALO_N, INT32_MAX], np.int64)
    got = rule_locators(ids, HALO_SPLIT, HALO_MY, HALO_N)
    assert got.tolist() == [4_999, -1, -5_000, 0, 4_998, -10_000, -HALO_N, 4_999, 4_999]
    every = np.arange(HALO_N)
    assert (rule_locators(every, HALO_SPLIT, HALO_MY, HALO_N) < 0).sum() == halo_remote()


def test_int8_oracle_is_vectorised_and_writes_every_byte():
    """The GPU file uses oracle.int8_rows as it is (it is already vectorised): its layout for F % 4 != 0, where the scale
    sits at round_up(F, 4), not at F."""
    x = np.array([[1.0, -2.0, 0.5, 127.0, -127.0]], np.float32)
    rows = int8_rows.quantize_rows(x)
    assert rows.shape == (1, 16)
    assert rows[0, 8:12].view("<f4")[0] == np.float32(127.0) / np.float32(127)
    assert (rows[0, 5:8] == 0).all() and (rows[0, 12:] == 0).all()


def test_rmat_degrees_ref_equals_the_oracle():
    for scale, n, ef in ((10, 1024, 6.0), (11, 1500, 3.0), (9, 300, 40.0)):
        indptr, _ = ormat.rmat_csr(scale, n, ef, seed=3)
        assert np.array_equal(rmat_degrees_ref(scale, n, ef, 3), np.diff(indptr))


def test_bf16_rule_restates_the_source():
    src = _source("gather.cu")
    body = re.search(r"uint32_t f32_to_bf16_rne\(float x\) \{(.*?)\n\}", src, re.S).group(1)
    assert "if ((u & 0x7fffffffu) > 0x7f800000u) return (u >> 16) | 0x40u;" in body
    assert "return (u + 0x7fffu + ((u >> 16) & 1u)) >> 16;" in body
    x = bf16_special_values()
    got = bf16_bits(x)
    finite = ~np.isnan(x)
    want = torch.from_numpy(x[finite].copy()).to(torch.bfloat16).view(torch.int16).numpy().view(np.uint16)
    assert np.array_equal(got[finite], want)                                 # round to nearest even, as torch rounds
    back = (got.astype(np.uint32) << 16).view(np.float32)
    assert np.array_equal(np.isnan(back), np.isnan(x))                       # NaN stays NaN (0x7F800001 too)
    assert np.array_equal(np.signbit(back), np.signbit(x))
    assert got[x.view(np.uint32) == 0x7F800001][0] == 0x7FC0 and got[x.view(np.uint32) == 0xFF800001][0] == 0xFFC0
    assert got[x.view(np.uint32) == 0x7F7FFFFF][0] == 0x7F80 and got[x.view(np.uint32) == 0xFF7FFFFF][0] == 0xFF80
    rs = np.random.RandomState(8)
    y = rs.randn(10_000).astype(np.float32) * np.float32(10.0) ** rs.randint(-40, 39, size=10_000).astype(np.float32)
    want = torch.from_numpy(y).to(torch.bfloat16).view(torch.int16).numpy().view(np.uint16)
    assert np.array_equal(bf16_bits(y), want)
