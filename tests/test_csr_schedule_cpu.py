"""The Python mirror of the hub / short row schedule of graphsage_b200/csrc/csr_rows.cuh, the stress cases that
test_zz_gpu_csr_schedule.py runs on it, and the checks that keep both honest: the mirror's constants equal the header's,
every case reaches the regimes it is built for on an H100 PCIe (114 SMs) and an H100 SXM (132 SMs), and the vectorised
max-backward reference equals oracle.full_neighbor_grad.max_backward.

The schedule: output rows with more than LONG entries go to the hub role, whose work item is (chunk of CHUNK rows, slice
of COLS columns); at most HUB_CAP * SMs hub CTAs, each looping over items with stride hub_blocks.  Every other row goes to
the short role, one warp per (row, slice of 32 V columns); at most SHORT_CAP * SMs CTAs of WARPS warps, each warp looping
with stride (short CTAs * WARPS).  A case only tests those loops if it makes them loop, so every case computes the regime
it reaches (`regime`) and asserts it (`require`).  Sizes come from the SM count, so a case cannot pass vacuously on a GPU
with more SMs.  Output rows are listed through `rows` (a few hundred nodes, many times over), so the grid regimes need no
big graph; gs_csr_max_backward has no `rows`, so its case is a real graph of 512 * SMs * 1.1 nodes."""
import math
import os
import re

import numpy as np
import pytest

from oracle import full_neighbor as fn
from oracle import full_neighbor_grad as fg

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "graphsage_b200", "csrc",
                      "csr_rows.cuh")

# ---------------------------------------------------------------- the mirror of csr_rows.cuh
THREADS = 256            # kCsrThreads
WARPS = THREADS // 32
LONG = 256               # kCsrLong: rows with more entries are hub rows
CHUNK = 256              # kHubChunk: rows per hub work item
COLS = 32                # kHubCols: columns per hub work item
PER_WARP = 8             # kHubPerWarp: a hub round is PER_WARP * WARPS = 64 entries
HUB_CAP = 4              # hub_blocks <= HUB_CAP * SMs
SHORT_CAP = 8 * 64       # short CTAs <= SHORT_CAP * SMs
UNROLL = {1: 8, 4: 8, 8: 4}   # the short role's loads in flight, by V (csr_aggregate_kernel; the max backward: V 1, 8)
SM_COUNTS = (114, 132)   # H100 PCIe, H100 SXM

HUB_DEGREES = (257, 320, 321, 384, 447, 448, 449, 1000, 4097)
SHORT_DEGREES = (0, 1, 3, 4, 5, 7, 8, 9, 63, 64, 65, 255, 256)
IN_DEGREES = (63, 64, 65, 255, 256) + HUB_DEGREES     # the transposed rows' (in-degree) counts placed on purpose
BIG = 100_000


def pad_cols(f):
    return (int(f) + 7) // 8 * 8


def csr_grid(rows, hub_slices, slices, sms):
    """csr_grid: (hub_items, hub_blocks, short_blocks)."""
    hub_items = -(-rows // CHUNK) * hub_slices
    return hub_items, min(hub_items, HUB_CAP * sms), min((rows * slices + WARPS - 1) // WARPS, SHORT_CAP * sms)


def regime(cnt, hub_slices, slices, sms, F, out_cols):
    """What a launch over output rows with cnt[i] entries reaches: hub items per hub CTA (rounds), the chunks holding hub
    rows, the most hub-bearing items one hub CTA takes, the short role's rounds, and whether a hub slice lies wholly past
    F (its lanes all have col_ok false and must still write zeros)."""
    cnt = np.asarray(cnt, np.int64)
    rows = len(cnt)
    hub_items, hub_blocks, short_blocks = csr_grid(rows, hub_slices, slices, sms)
    chunks = np.unique(np.nonzero(cnt > LONG)[0] // CHUNK)
    items = (chunks[:, None] * hub_slices + np.arange(hub_slices)).ravel()
    per_cta = np.bincount(items % hub_blocks, minlength=hub_blocks) if len(items) else np.zeros(1, np.int64)
    return dict(rows=rows, hub_items=hub_items, hub_blocks=hub_blocks, hub_rounds=-(-hub_items // hub_blocks),
                hub_chunks=len(chunks), n_chunks=-(-rows // CHUNK),
                last_chunk_hub=bool(len(chunks)) and int(chunks[-1]) == -(-rows // CHUNK) - 1,
                hub_items_per_cta=int(per_cta.max()),
                short_rounds=-(-rows * slices // (short_blocks * WARPS)),
                dead_slice=(hub_slices - 1) * COLS >= F and out_cols > (hub_slices - 1) * COLS,
                counts=set(np.unique(cnt).tolist()))


def describe(reg):
    return ("%d rows: %d hub items on %d hub CTAs (%d rounds, up to %d items with hub rows per CTA), hub rows in %d of %d "
            "chunks (last: %s), %d short-role rounds%s" % (
                reg["rows"], reg["hub_items"], reg["hub_blocks"], reg["hub_rounds"], reg["hub_items_per_cta"],
                reg["hub_chunks"], reg["n_chunks"], "yes" if reg["last_chunk_hub"] else "no", reg["short_rounds"],
                ", a hub slice wholly past F" if reg["dead_slice"] else ""))


def require(reg, dead_slice=False, counts=()):
    """The regimes every case must reach (and, where asked, a hub slice wholly past F and the given row lengths)."""
    what = describe(reg)
    assert reg["hub_items"] > 2 * reg["hub_blocks"], what
    assert reg["hub_items_per_cta"] >= 2, what              # some hub CTA computes hub rows on a second item
    assert reg["hub_chunks"] >= 3 and reg["last_chunk_hub"], what
    assert reg["short_rounds"] >= 2, what
    assert reg["rows"] % CHUNK != 0, what                   # the last chunk is partial
    if dead_slice:
        assert reg["dead_slice"], what
    missing = set(counts) - reg["counts"]
    assert not missing, "row lengths %s never occur: %s" % (sorted(missing), what)
    return what


def rows_for(hub_slices, slices, sms):
    """An output row count that makes hub_items > 2 * HUB_CAP * SMs and rows * slices > WARPS * SHORT_CAP * SMs, 10 %
    over, with a partial last chunk."""
    need = max((2 * HUB_CAP * sms // hub_slices + 1) * CHUNK, WARPS * SHORT_CAP * sms // slices + 1)
    return int(need * 1.1) // CHUNK * CHUNK + 77


# ---------------------------------------------------------------- gs_csr_aggregate's launches
LAYOUT_V = {"fp32": 4, "fp32_odd": 1, "bf16": 8}      # a 16-byte pitch (float4), an odd pitch (scalar), bf16 (8 x bf16)


def out_pitch(layout, F, wide):
    """The out= pitch: pad_cols(F), or wider by 32 columns (33 for the odd layout: an odd pitch) - then the last hub
    slice lies wholly past F."""
    return pad_cols(F) + ((33 if layout == "fp32_odd" else 32) if wide else 0)


def aggregate_slices(layout, pitch):
    """(hub_slices, short slices) of gs_csr_aggregate for an out pitch: ceil(pitch / 32), ceil(pitch / (32 V))."""
    V = LAYOUT_V[layout]
    return -(-pitch // COLS), -(-pitch // (32 * V))


N_AGG = 300


def _duplicates_and_self_loops(indptr, indices):
    deg = np.diff(indptr)
    for i in np.nonzero(deg >= 2)[0][::4]:                  # every fourth row repeats its first entry
        indices[indptr[i] + 1] = indices[indptr[i]]
    for i in np.nonzero(deg >= 1)[0][1::9]:                 # self loops
        indices[indptr[i + 1] - 1] = i


def stress_graph(rs, big=True):
    """(indptr, indices, n_src) over N_AGG nodes: each SHORT_DEGREES degree on two nodes, each HUB_DEGREES degree on one,
    one row of BIG entries (or 600 without big), random degrees below 70 elsewhere.  Entries in [0, n_src) with 2 % out
    of range (-1, -7, n_src, n_src + 3: the dummy row), duplicates and self loops."""
    n, n_src = N_AGG, N_AGG + 40
    deg = rs.randint(0, 70, size=n)
    deg[:2 * len(SHORT_DEGREES)] = SHORT_DEGREES * 2
    hubs = rs.choice(np.arange(2 * len(SHORT_DEGREES), n), len(HUB_DEGREES) + 1, replace=False)
    deg[hubs[:-1]] = HUB_DEGREES
    deg[hubs[-1]] = BIG if big else 600
    indptr = np.concatenate([[0], np.cumsum(deg)]).astype(np.int64)
    indices = rs.randint(0, n_src, size=int(indptr[-1])).astype(np.int32)
    bad = rs.rand(len(indices)) < 0.02
    indices[bad] = rs.choice([-1, -7, n_src, n_src + 3], size=int(bad.sum()))
    _duplicates_and_self_loops(indptr, indices)
    return indptr, indices, n_src


def stress_rows(rs, cnt, n_rows, outside=()):
    """int32 [n_rows] node ids for `rows`: short nodes (cnt <= LONG) everywhere; hub nodes by chunk - none, one, two or
    three per chunk in a repeating pattern, one chunk with the same hub three times, one in the last partial chunk - the
    node with the most entries once, in the middle chunk; 0.3 % of the ids from `outside` (ids outside [0, N))."""
    cnt = np.asarray(cnt)
    short = np.nonzero(cnt <= LONG)[0]
    top = int(np.argmax(cnt))
    hubs = np.setdiff1d(np.nonzero(cnt > LONG)[0], [top])
    rows = rs.choice(short, n_rows).astype(np.int64)
    if len(outside):
        out = rs.rand(n_rows) < 0.003
        rows[out] = rs.choice(np.asarray(outside), int(out.sum()))
    n_chunks = -(-n_rows // CHUNK)
    per = np.array([0, 1, 0, 2, 0, 0, 3, 1])[np.arange(n_chunks) % 8]
    per[-1] = max(per[-1], 1)
    for k in np.nonzero(per)[0]:
        lo = k * CHUNK
        at = lo + rs.choice(min(CHUNK, n_rows - lo), per[k], replace=False)
        rows[at] = rs.choice(hubs, per[k])
    k = n_chunks // 3
    rows[k * CHUNK + rs.choice(CHUNK, 3, replace=False)] = hubs[0]
    rows[(n_chunks // 2) * CHUNK + 17] = top
    return rows.astype(np.int32)


def node_counts(indptr, ids):
    """Entries of each id's row; 0 for an id outside [0, N)."""
    indptr = np.asarray(indptr, np.int64)
    ids = np.asarray(ids, np.int64)
    n = len(indptr) - 1
    ok = (ids >= 0) & (ids < n)
    safe = np.where(ok, ids, 0)
    return np.where(ok, indptr[safe + 1] - indptr[safe], 0)


# op, layout, F, wide out=: each op and each layout meets every F once; F <= 33 runs on a wide out=, F = 602 (one case
# per op and per layout) carries the BIG row
AGG_CASES = [("mean", "fp32", 602, False), ("mean", "fp32_odd", 33, True), ("mean", "bf16", 5, True),
             ("mean_self", "fp32", 33, True), ("mean_self", "fp32_odd", 5, True), ("mean_self", "bf16", 602, False),
             ("max", "fp32", 5, True), ("max", "fp32_odd", 602, False), ("max", "bf16", 33, True)]
# op, rate, layout, F, wide: the masked means, without the BIG row (their oracle runs Philox per entry)
MASK_CASES = [("mean", 0.1, "fp32", 602, False), ("mean", 0.5, "bf16", 33, True),
              ("mean_self", 0.1, "fp32_odd", 5, True), ("mean_self", 0.5, "bf16", 602, False)]


def aggregate_case(sms, layout, F, wide, big, seed):
    """The stress graph, its rows and their regime for one gs_csr_aggregate case."""
    rs = np.random.RandomState(seed)
    indptr, indices, n_src = stress_graph(rs, big)
    pitch = out_pitch(layout, F, wide)
    hub_slices, slices = aggregate_slices(layout, pitch)
    n = len(indptr) - 1
    rows = stress_rows(rs, np.diff(indptr), rows_for(hub_slices, slices, sms), outside=(-1, -5, n, n + 7, n + 100))
    reg = regime(node_counts(indptr, rows), hub_slices, slices, sms, F, pitch)
    return dict(indptr=indptr, indices=indices, n_src=n_src, rows=rows, pitch=pitch, regime=reg)


def aggregate_row_counts(layout):
    """The row lengths an aggregate case must contain: every short degree (the kUnroll edges of its V among them) and
    every hub degree."""
    V = LAYOUT_V[layout]
    u = UNROLL[V]
    return set(SHORT_DEGREES) | set(HUB_DEGREES) | {u - 1, u, u + 1}


# ---------------------------------------------------------------- graphs with placed in- and out-degrees
def spread_nodes(rs, n_rows, k, period=0):
    """k distinct rows spread over the chunks of n_rows rows past chunk 0: four share one chunk, one is in the last
    (partial) chunk but is not its last row (the dummy row), the rest are in distinct chunks.  With a period, one of them
    is `period` chunks after the shared chunk: a hub CTA whose stride is `period` chunks takes both."""
    n_chunks = -(-n_rows // CHUNK)
    assert n_chunks - 2 >= k - 4 + (period > 0) and n_rows % CHUNK >= 8
    c0 = rs.randint(1, n_chunks - 1 - period)
    rest = np.setdiff1d(np.arange(1, n_chunks - 1), [c0, c0 + period])
    chunks = np.concatenate([[c0 + period] if period else [], rs.choice(rest, k - 5 - (period > 0), replace=False)])
    nodes = list(c0 * CHUNK + rs.choice(CHUNK, 4, replace=False))
    nodes += list(chunks.astype(np.int64) * CHUNK + rs.randint(0, CHUNK, size=k - 5))
    nodes += [(n_chunks - 1) * CHUNK + rs.randint(0, n_rows % CHUNK - 1)]
    assert len(set(nodes)) == k
    return rs.permutation(np.array(nodes, np.int64))


def degree_graph(rs, n, out_deg, in_deg, n_bad):
    """Forward CSR over n nodes with out_deg[i] entries in row i and exactly in_deg[v] entries equal to v for the nodes of
    in_deg (a dict); the other entries are uniform over the other nodes, n_bad of them out of range (-1, -7, n + 1, n + 5:
    the dummy row).  Rows get duplicates and self loops by swapping entries between rows, which keeps every in-degree."""
    out_deg = np.asarray(out_deg, np.int64)
    placed = np.fromiter(in_deg.keys(), np.int64)
    fixed = np.repeat(placed, np.fromiter(in_deg.values(), np.int64))
    rest = int(out_deg.sum()) - len(fixed) - n_bad
    assert rest > 0
    others = np.setdiff1d(np.arange(n), placed)
    dst = np.concatenate([fixed, rs.choice(others, rest), rs.choice([-1, -7, n + 1, n + 5], n_bad)])
    rs.shuffle(dst)
    indptr = np.concatenate([[0], np.cumsum(out_deg)]).astype(np.int64)
    row_of = np.repeat(np.arange(n), out_deg)
    two = np.nonzero(out_deg >= 2)[0]
    for k, i in enumerate(rs.choice(two, min(400, len(two)), replace=False)):
        lo = indptr[i]
        v = i if k % 2 else dst[lo]                          # a self loop, or a duplicate of the row's first entry
        at = np.nonzero((dst == v) & (row_of != i))[0]
        if len(at):
            p = at[rs.randint(len(at))]
            dst[p], dst[lo + 1] = dst[lo + 1], dst[p]
    return indptr, dst.astype(np.int32)


N_SUM = 5000


def sum_graph(rs):
    """A forward CSR over N_SUM nodes whose transpose has in-degree hubs spread over its chunks (IN_DEGREES placed by
    spread_nodes) and a dummy row N with more than 256 entries (300 empty rows and 1 % out-of-range entries)."""
    n = N_SUM
    out_deg = rs.randint(1, 12, size=n)
    out_deg[rs.choice(n, 300, replace=False)] = 0
    nodes = spread_nodes(rs, n + 1, len(IN_DEGREES))
    return degree_graph(rs, n, out_deg, dict(zip(nodes.tolist(), IN_DEGREES)), int(0.01 * out_deg.sum()))


# plain: layout, F, wide; masked: with_self, layout, F, wide
SUM_CASES = [("fp32", 602, False), ("fp32_odd", 5, True)]
MASKED_SUM_CASES = [(False, "fp32", 33, True), (True, "fp32_odd", 70, False)]


def sum_case(sms, layout, F, wide, with_self, seed):
    """The sum graph, its transpose (with slots) and rows over the transposed rows with their regime."""
    rs = np.random.RandomState(seed)
    indptr, indices = sum_graph(rs)
    t_indptr, t_indices, t_slot = transpose_slots(indptr, indices, with_self)
    pitch = out_pitch(layout, F, wide)
    hub_slices, slices = aggregate_slices(layout, pitch)
    rows = stress_rows(rs, np.diff(t_indptr), rows_for(hub_slices, slices, sms))
    reg = regime(node_counts(t_indptr, rows), hub_slices, slices, sms, F, pitch)
    return dict(indptr=indptr, indices=indices, t_indptr=t_indptr, t_indices=t_indices, t_slot=t_slot, rows=rows,
                pitch=pitch, regime=reg, natural=regime(np.diff(t_indptr), hub_slices, slices, sms, F, pitch))


BWD_F = 256


def backward_graph(rs, sms, F=BWD_F):
    """A forward CSR for gs_csr_max_backward whose N + 1 rows make both phases loop on an H100 with `sms` SMs: forward hubs
    (HUB_DEGREES, phase a) and in-degree hubs (IN_DEGREES, phase b) placed by spread_nodes, every SHORT_DEGREES degree on
    four nodes, 300 empty rows and 1 % out-of-range entries (the dummy row's transposed row is a hub), degrees 1 .. 3
    elsewhere."""
    slices = -(-F // COLS)
    n = int(WARPS * SHORT_CAP * sms // slices * 1.1) // CHUNK * CHUNK + 140
    out_deg = rs.randint(1, 4, size=n)
    out_deg[rs.choice(n, 300, replace=False)] = 0
    out_deg[rs.choice(n, 4 * len(SHORT_DEGREES), replace=False)] = SHORT_DEGREES * 4
    period = HUB_CAP * sms // slices                       # the hub CTAs' stride in chunks
    out_deg[spread_nodes(rs, n + 1, len(HUB_DEGREES), period)] = HUB_DEGREES
    in_nodes = spread_nodes(rs, n + 1, len(IN_DEGREES), period)
    return degree_graph(rs, n, out_deg, dict(zip(in_nodes.tolist(), IN_DEGREES)), int(0.01 * out_deg.sum()))


def backward_case(sms, seed, F=BWD_F):
    """The max-backward graph, its effective CSR and transpose, and both phases' regimes."""
    rs = np.random.RandomState(seed)
    indptr, indices = backward_graph(rs, sms, F)
    eptr, eidx = effective_csr(indptr, indices)
    t_indptr, t_indices = transpose(eptr, eidx)
    slices = -(-F // COLS)
    return dict(indptr=indptr, indices=indices, eptr=eptr, eidx=eidx, t_indptr=t_indptr, t_indices=t_indices,
                regime_a=regime(np.diff(eptr), slices, slices, sms, F, F),
                regime_b=regime(np.diff(t_indptr), slices, slices, sms, F, F))


# ---------------------------------------------------------------- vectorised order-exact references
def effective_csr(indptr, indices, with_self=False):
    """oracle.full_neighbor_grad.effective_csr without its per-row loop: (eptr [N + 2], eidx) int64."""
    indptr = np.asarray(indptr, np.int64)
    indices = np.asarray(indices, np.int64)
    N = len(indptr) - 1
    deg = np.maximum(np.diff(indptr), 0)
    cnt = np.concatenate([np.maximum(deg, 1), [1]]) + (1 if with_self else 0)
    eptr = np.concatenate([[0], np.cumsum(cnt)]).astype(np.int64)
    eidx = np.full(int(eptr[-1]), N, np.int64)
    row = np.repeat(np.arange(N), deg)
    off = np.arange(len(row)) - np.repeat(indptr[:-1], deg)
    e = indices[np.repeat(indptr[:-1], deg) + off]
    eidx[eptr[row] + off] = np.where((e < 0) | (e > N), N, e)
    if with_self:
        eidx[eptr[1:] - 1] = np.arange(N + 1)
    return eptr, eidx


def transpose(eptr, eidx):
    """oracle.full_neighbor_grad.csr_transpose from an effective CSR: (t_indptr [N + 2], t_indices) int64."""
    src = np.repeat(np.arange(len(eptr) - 1), np.diff(eptr))
    order = np.argsort(eidx, kind="stable")
    t_indptr = np.concatenate([[0], np.cumsum(np.bincount(eidx, minlength=len(eptr) - 1))]).astype(np.int64)
    return t_indptr, src[order].astype(np.int64)


def transpose_slots(indptr, indices, with_self=False):
    """oracle.full_neighbor_dropout.csr_transpose_slots without its per-row loop: (t_indptr, t_indices, t_slot)."""
    eptr, eidx = effective_csr(indptr, indices, with_self)
    ecnt = np.diff(eptr)
    src = np.repeat(np.arange(len(ecnt)), ecnt)
    slot = np.arange(len(eidx)) - eptr[src]
    raw = np.concatenate([np.maximum(np.diff(np.asarray(indptr, np.int64)), 0), [0]])[src]
    slot = np.where(with_self & (slot == ecnt[src] - 1), -2, np.where(raw > 0, slot, -1))
    order = np.argsort(eidx, kind="stable")
    t_indptr, _ = transpose(eptr, eidx)
    return t_indptr, src[order].astype(np.int64), slot[order].astype(np.int64)


def _by_position(ptr, idx):
    """(order, steps): the rows sorted by length, longest first, and for t = 0, 1, ... the pair (k, entry t of each of the
    first k sorted rows), k the number of rows with more than t entries - so a row's entries come in CSR order and the
    rows that have one are a prefix of `order`."""
    cnt = np.diff(ptr)
    order = np.argsort(-cnt, kind="stable")
    desc, start = -cnt[order], ptr[order]

    def steps():
        for t in range(int(cnt.max()) if len(cnt) else 0):
            k = int(np.searchsorted(desc, -t))
            yield k, idx[start[:k] + t]
    return order, steps()


def _unsort(order, x):
    out = np.empty_like(x)
    out[order] = x
    return out


def row_max(z, eptr, eidx):
    """The max of z over each effective row: csr_aggregate's "max" over the N + 1 rows (no NaN, so in any order)."""
    z = np.asarray(z, np.float32)
    order, steps = _by_position(eptr, eidx)
    m = np.full((len(order), z.shape[1]), -np.inf, np.float32)
    for k, j in steps:
        m[:k] = np.fmax(m[:k], z[j])
    return _unsort(order, m)


def max_backward(z, m, dm, eptr, eidx, t_indptr, t_indices):
    """oracle.full_neighbor_grad.max_backward, bit for bit, vectorised over rows: (s, dz) fp32 [N + 1, F].  The tie counts
    of phase (a) are integers, exact in fp32 in any order; the sums of phase (b) run in transposed order."""
    z, m, dm = (np.asarray(x, np.float32) for x in (z, m, dm))
    order, steps = _by_position(eptr, eidx)
    mo, cnt = m[order], np.zeros_like(m)
    for k, j in steps:
        cnt[:k] += z[j] == mo[:k]
    with np.errstate(divide="ignore", invalid="ignore"):
        s = (dm / _unsort(order, cnt)).astype(np.float32)
    order, steps = _by_position(t_indptr, t_indices)
    zo, acc = z[order], np.zeros_like(z)
    for k, i in steps:
        a = acc[:k]
        acc[:k] = np.where(zo[:k] == m[i], a + s[i], a)
    return s, _unsort(order, np.where(zo > 0, acc, np.float32(0)))


# ---------------------------------------------------------------- the checks
def _header():
    with open(HEADER) as f:
        return f.read()


def test_mirror_constants_equal_the_header():
    src = _header()

    def const(name):
        got = re.findall(r"constexpr\s+\w+\s+%s\s*=\s*(\d+)\s*;" % name, src)
        assert len(got) == 1, name
        return int(got[0])
    assert const("kCsrThreads") == THREADS
    assert const("kCsrLong") == LONG
    assert const("kHubChunk") == CHUNK
    assert const("kHubCols") == COLS
    assert const("kHubPerWarp") == PER_WARP
    grid = re.search(r"inline unsigned csr_grid\(.*?\n}", src, re.S).group(0)

    def cap(lhs):
        got = re.findall(r"%s\s*=\s*std::min<int64_t>\((.*)\);" % lhs, grid)
        assert len(got) == 1, lhs
        factors = re.fullmatch(r".*\(int64_t\)sm_count\(\)((?:\s*\*\s*\d+)+)", got[0].strip())
        assert factors, got[0]
        return math.prod(int(x) for x in re.findall(r"\d+", factors.group(1)))
    assert cap("hub_blocks") == HUB_CAP
    assert cap("const int64_t short_blocks") == SHORT_CAP
    assert "(rows + kHubChunk - 1) / kHubChunk * hub_slices" in grid
    assert "(rows * slices + 7) / 8" in grid
    here = os.path.dirname(HEADER)
    with open(os.path.join(here, "csr_aggregate.cu")) as f:
        agg = f.read()
    with open(os.path.join(here, "csr_backward.cu")) as f:
        bwd = f.read()
    assert "csr_rows<V, V == 8 ? 4 : 8>" in agg                    # UNROLL[8] = 4, UNROLL[4] = UNROLL[1] = 8
    assert "csr_rows<1, 8>" in bwd
    assert "a.n_slices = (int32_t)((out_pitch + 32 * V - 1) / (32 * V));" in agg
    assert "a.hub_slices = (int32_t)((out_pitch + kHubCols - 1) / kHubCols);" in agg


def test_csr_grid_mirror():
    assert csr_grid(1, 19, 5, 132) == (19, 19, 1)
    assert csr_grid(257, 1, 1, 132) == (2, 2, 33)
    assert csr_grid(10 ** 6, 2, 1, 132) == (3907 * 2, 528, 67584)
    reg = regime([0] * 254 + [300] * 3 + [0] * 300, 1, 1, 132, 5, 8)
    assert reg["hub_chunks"] == 2 and not reg["last_chunk_hub"] and reg["short_rounds"] == 1
    assert reg["hub_items"] == 3 and reg["hub_items_per_cta"] == 1 and not reg["dead_slice"]
    reg = regime([300] * 2000, 2, 1, 1, 5, 40)
    assert reg["hub_blocks"] == 4 and reg["hub_items_per_cta"] == 4 and reg["last_chunk_hub"] and reg["dead_slice"]
    assert not regime([300] * 2000, 2, 1, 1, 33, 40)["dead_slice"]


@pytest.mark.parametrize("sms", SM_COUNTS)
@pytest.mark.parametrize("op,layout,F,wide", AGG_CASES)
def test_aggregate_cases_reach_every_regime(sms, op, layout, F, wide):
    c = aggregate_case(sms, layout, F, wide, F == 602, seed=F)
    require(c["regime"], dead_slice=wide, counts=aggregate_row_counts(layout) | ({BIG} if F == 602 else {600}))
    assert not c["regime"]["dead_slice"] or wide


@pytest.mark.parametrize("sms", SM_COUNTS)
@pytest.mark.parametrize("op,p,layout,F,wide", MASK_CASES)
def test_masked_cases_reach_every_regime(sms, op, p, layout, F, wide):
    c = aggregate_case(sms, layout, F, wide, False, seed=F + 1)
    require(c["regime"], dead_slice=wide, counts=aggregate_row_counts(layout))


@pytest.mark.parametrize("sms", SM_COUNTS)
@pytest.mark.parametrize("with_self,layout,F,wide", [(None,) + c for c in SUM_CASES] + MASKED_SUM_CASES)
def test_sum_cases_reach_every_regime(sms, with_self, layout, F, wide):
    c = sum_case(sms, layout, F, wide, bool(with_self), seed=F + 2)
    extra = 1 if with_self else 0
    require(c["regime"], dead_slice=wide, counts={d + extra for d in IN_DEGREES})
    t_cnt = np.diff(c["t_indptr"])
    assert t_cnt[-1] > LONG                                          # the dummy row N is a hub
    assert c["natural"]["hub_chunks"] >= 3 and c["natural"]["last_chunk_hub"]
    if with_self:                                                    # hub rows carry -1 (the dummy's) and -2 slots
        hub_slots = np.concatenate([c["t_slot"][c["t_indptr"][j]:c["t_indptr"][j + 1]] for j in np.nonzero(t_cnt > LONG)[0]])
        assert (hub_slots == -1).any() and (hub_slots == -2).sum() == (t_cnt > LONG).sum()


@pytest.mark.parametrize("sms", SM_COUNTS)
def test_max_backward_case_reaches_every_regime(sms):
    c = backward_case(sms, seed=5)
    require(c["regime_a"], counts=set(SHORT_DEGREES[1:]) | set(HUB_DEGREES) | {1})
    require(c["regime_b"], counts=set(IN_DEGREES))
    assert np.diff(c["t_indptr"])[-1] > LONG


def _small_graph(rs, n=150):
    out_deg = rs.randint(0, 9, size=n)
    out_deg[[5, 77, 140]] = [300, 270, 600]
    return degree_graph(rs, n, out_deg, {3: 290, 100: 64, 149: 257}, 30)


@pytest.mark.parametrize("with_self", [False, True])
def test_vectorised_transposes_equal_the_oracle(with_self):
    from oracle import full_neighbor_dropout as fd
    rs = np.random.RandomState(11)
    indptr, indices = _small_graph(rs)
    eptr, eidx = effective_csr(indptr, indices, with_self)
    want_ptr, want_idx = fg.effective_csr(indptr, indices, with_self)
    assert np.array_equal(eptr, want_ptr) and np.array_equal(eidx, want_idx)
    got = transpose_slots(indptr, indices, with_self)
    for a, b in zip(got, fd.csr_transpose_slots(indptr, indices, with_self)):
        assert np.array_equal(a, b)
    assert all(np.array_equal(a, b) for a, b in zip(transpose(eptr, eidx), fg.csr_transpose(indptr, indices, with_self)))


def test_degree_graph_places_its_degrees():
    rs = np.random.RandomState(4)
    indptr, indices = _small_graph(rs)
    assert np.diff(indptr)[[5, 77, 140]].tolist() == [300, 270, 600]
    assert [(indices == v).sum() for v in (3, 100, 149)] == [290, 64, 257]
    assert ((indices < 0) | (indices > 150)).sum() == 30
    assert any(i in indices[indptr[i]:indptr[i + 1]] for i in range(150))                     # self loops
    assert any(len(set(indices[a:b])) < b - a for a, b in zip(indptr[:-1], indptr[1:]))      # duplicates


@pytest.mark.parametrize("F", [1, 7, 40])
def test_vectorised_max_backward_equals_the_oracle(F):
    rs = np.random.RandomState(F)
    indptr, indices = _small_graph(rs)
    z = rs.randint(0, 4, size=(151, F)).astype(np.float32)
    dm = rs.randn(151, F).astype(np.float32)
    eptr, eidx = effective_csr(indptr, indices)
    m = row_max(z, eptr, eidx)
    assert np.array_equal(m.view(np.uint32), fn.csr_aggregate(z, indptr, indices, "max").view(np.uint32))
    want_s, want_dz = fg.max_backward(z, m, dm, indptr, indices)
    s, dz = max_backward(z, m, dm, eptr, eidx, *transpose(eptr, eidx))
    assert np.array_equal(s.view(np.uint32), want_s.view(np.uint32))
    assert np.array_equal(dz.view(np.uint32), want_dz.view(np.uint32))
    assert (dz != 0).any() and (z == 0).any()
