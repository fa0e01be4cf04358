"""Fixed-fanout neighbour draws in proportion to edge weight: the contract of gs_csr_alias_build, gs_sample_alias and
gs_sample_alias_khop (ops.csr_alias_table / sample_alias / sample_alias_khop, WeightedNeighborSampler).  Plain numpy,
in the kernels' order, bit for bit.

Weights w are float32, one per entry of `indices`, aligned with it; they are data (no gradient flows to them).

Eligibility (as oracle/weighted_sampling.py): an entry with finite w > 0 is eligible; NaN, zero and negative weights are
never drawn.  A row with any +inf entry draws uniformly among its +inf entries (the limit of proportional sampling): its
+inf entries count as weight 1 and every other entry as ineligible.  A row with no eligible entry - an empty row
included - draws the dummy node N = len(indptr) - 1, and so does a query id outside [0, N) (N itself included).

Masses.  Row v has d entries (d < 2^31; the build refuses longer rows), T = d 2^32 and n_e >= 1 eligible entries with
weights w_j (the +inf rule applied).  All fp64 operations below are IEEE round-to-nearest, never contracted:
  S    = the fp64 sum of the eligible w_j (widened exactly from fp32), one addition at a time in ascending CSR order;
  R    = T - n_e (one unit per eligible entry is reserved: that pays for the floor m_j >= 1);
  x_j  = fl(fl(w_j / S) * fl(R)),  b_j = min(floor(min(x_j, fl(R))), R)  (uint64);
  rem  = R - sum_j b_j  (exact, signed);
  rem >= 0: eligible entry of rank r (0-based, CSR order among the eligible) gets share_j = rem // n_e + (r < rem % n_e);
  rem <  0: the units are taken greedily in CSR order: take_j = min(b_j, max(0, -rem - sum_{i<j} b_i));
  m_j  = 1 + b_j + share_j - take_j for an eligible entry, 0 for an ineligible one.
So sum_j m_j = T exactly, every eligible m_j >= 1 and every ineligible m_j = 0.  With u = 2^-53, each rounding above is
within u relatively and S within (n_e - 1) u of the exact sum, so |b_j - w_j R / S| <= 1 + 4u w_j R / S + ...,
|rem| <= n_e + (n_e + 5) u R, and
  |m_j - w_j T / S| <= n_e + 3 + (n_e + 8) 2^-53 T            (alias_mass_bound states it; the tests check it exactly).
In probability terms: |m_j / T - w_j / S| <= (n_e + 3) / T + (n_e + 8) 2^-53, i.e. under 2^-31 + n_e 2^-53 for every row.

Buckets.  An integer sweep (the two-pointer form of Vose's method) turns the masses into d buckets of capacity C = 2^32.
Entries with m < C are light, entries with m >= C heavy; a light pointer i and a heavy pointer j each move through the
row in ascending position, w holds the current heavy's remaining mass:
  i = first light, j = first heavy, w = m_j
  while j < d:
    w > C:  bucket i = (thr m_i, id_i, alias id_j); w -= C - m_i; i = next light
    w == C: bucket j = (thr 0, id_j, alias id_j) - a full bucket aliases itself; j = next heavy, w = m_j
    w < C:  j' = next heavy; bucket j = (thr w, id_j, alias id_j'); w = m_j' - (C - w); j = j'
Mass is conserved, so every light is served before the heavies run out and the last heavy ends full.  A row whose masses
are all C (equal weights) is all full buckets.  A row with no eligible entry gets (0, N, N) records.
Record b of row v lives at table[indptr[v] + b] = (thr, id, alias, 0) as four 32-bit words (16 bytes per CSR entry).

Draw.  Draw j (0 <= j < k) of output position t (0 <= t < n) in a call with counter c:
  (r0, r1, r2, r3) = philox4x32_10((c_lo, c_hi, t, STREAM_ALIAS + (j >> 1)), split64(seed))
  (a, b) = (r0, r1) for even j, (r2, r3) for odd j
  bucket = mulhi32(a, d);  out = id_bucket if b < thr_bucket else alias_bucket.
The law of one draw from row v: P(u) = sum_b [id_b = u] thr_b + [alias_b = u] (C - thr_b), over T, taking the bucket
as uniform (alias_law, exact integers; it equals the masses summed by id).  mulhi32 gives bucket b probability
floor or ceil of 2^32 / d over 2^32, a relative bias of at most d / 2^32 on every bucket, so
  |P(u) - sum_{j: id_j = u} w_j / S| <= d 2^-32 + sum over those j of the mass bound above.
The sampled mean (1/k) sum_i x_{J_i} is therefore an unbiased estimator (up to these bounds) of sum_j (w_j / S) x_j.

k-hop.  A k-hop call with fanouts (k_0 .. k_{L-1}) and counter c is byte-identical to L single-hop calls with counters
c, c + 1, .., c + L - 1, each numbering its output positions t from 0.  A call advances the sampler's counter by 1, a
k-hop call by L (UniformNeighborSampler's rule).

Test infrastructure - not imported by the product.
"""
import numpy as np

from .philox import mulhi32, philox4x32_10, split64

STREAM_ALIAS = 0x90000000
CAP = 1 << 32
MAX_ROW = 1 << 31          # rows of 2^31 entries or more are refused


def _rows(indptr):
    indptr = np.asarray(indptr, dtype=np.int64)
    deg = np.maximum(indptr[1:] - indptr[:-1], 0)
    return indptr, deg


def eligibility(indptr, w):
    """(eligible bool [E], fp64 weight used [E]) after the +inf rule."""
    indptr, deg = _rows(indptr)
    w = np.asarray(w)
    if w.dtype != np.float32 or w.ndim != 1:
        raise ValueError("weights must be a 1-D float32 array, one value per CSR entry")
    E = len(w)
    seg = np.repeat(np.arange(len(deg)), deg)
    lo = int(indptr[0]) if len(indptr) else 0
    seg_full = np.full(E, -1, np.int64)
    seg_full[lo:lo + len(seg)] = seg
    with np.errstate(invalid="ignore"):
        fin = np.isfinite(w) & (w > 0)
    inf = np.isposinf(w)
    row_inf = np.zeros(len(deg) + 1, bool)
    row_inf[seg_full[inf]] = True
    row_inf[-1] = False                                     # entries outside every row (seg -1) are never drawn
    in_row = seg_full >= 0
    use_inf = row_inf[seg_full]
    elig = in_row & np.where(use_inf, inf, fin)
    wv = np.where(elig, np.where(use_inf, 1.0, w.astype(np.float64)), 0.0)
    return elig, wv, seg_full


def masses(indptr, w):
    """uint64 [E]: the integer mass m_j of every entry (the docstring's rule, vectorised)."""
    indptr, deg = _rows(indptr)
    N = len(deg)
    elig, wv, seg = eligibility(indptr, w)
    E = len(wv)
    m = np.zeros(E, np.uint64)
    if E == 0 or N == 0:
        return m
    ok = seg >= 0
    sg = seg[ok]
    S = np.zeros(N, np.float64)
    np.add.at(S, sg, wv[ok])                                # one addition at a time, in CSR order within each row
    ne = np.zeros(N, np.int64)
    np.add.at(ne, sg, elig[ok].astype(np.int64))
    T = deg.astype(np.uint64) << np.uint64(32)
    R = (T - ne.astype(np.uint64)).astype(np.int64)        # < 2^63
    Rf = R.astype(np.float64)
    e = ok & elig
    es = seg[e]
    with np.errstate(divide="ignore", invalid="ignore"):
        x = (wv[e] / S[es]) * Rf[es]
    x = np.minimum(x, Rf[es])
    b = np.zeros(E, np.int64)
    b[e] = np.minimum(np.floor(x).astype(np.uint64).astype(np.int64), R[es])
    sumb = np.zeros(N, np.int64)
    np.add.at(sumb, sg, b[ok])
    rem = R - sumb
    # rank among the eligible and the b prefix before each entry, within its row
    start = indptr[:-1]
    cnt_e = np.cumsum(elig.astype(np.int64))
    cnt_b = np.cumsum(b)
    pos = np.nonzero(ok)[0]
    first = start[sg]                                       # the row's first entry
    before_e = np.where(first > 0, cnt_e[np.maximum(first - 1, 0)], 0)
    before_b = np.where(first > 0, cnt_b[np.maximum(first - 1, 0)], 0)
    rank = cnt_e[pos] - before_e - 1
    pre_b = cnt_b[pos] - before_b - b[pos]
    r = rem[sg]
    n_e = ne[sg]
    safe_ne = np.maximum(n_e, 1)
    share = np.where(r >= 0, r // safe_ne + (rank < r % safe_ne), 0)
    take = np.where(r < 0, np.minimum(b[pos], np.maximum(0, -r - pre_b)), 0)
    mm = np.where(elig[pos], 1 + b[pos] + share - take, 0)
    m[pos] = mm.astype(np.uint64)
    return m


def sweep(m, ids, pad):
    """The bucket records (thr, id, alias) of one row from its masses (Python ints) and neighbour ids."""
    d = len(m)
    thr = [0] * d
    ida = [int(x) for x in ids]
    alias = list(ida)
    if d == 0:
        return thr, ida, alias
    if sum(m) == 0:
        return thr, [pad] * d, [pad] * d
    heavy = [x >= CAP for x in m]

    def nxt(p, want):
        while p < d and heavy[p] != want:
            p += 1
        return p

    i, j = nxt(0, False), nxt(0, True)
    w = m[j] if j < d else 0
    while j < d:
        if w > CAP:
            assert i < d, "mass not conserved"
            thr[i], alias[i] = m[i], ida[j]
            w -= CAP - m[i]
            i = nxt(i + 1, False)
        elif w == CAP:
            thr[j], alias[j] = 0, ida[j]
            j = nxt(j + 1, True)
            w = m[j] if j < d else 0
        else:
            j2 = nxt(j + 1, True)
            assert j2 < d, "mass not conserved"
            thr[j], alias[j] = w, ida[j2]
            w = m[j2] - (CAP - w)
            j = j2
    assert i >= d, "mass not conserved"
    return thr, ida, alias


def build_table(indptr, indices, w):
    """int32 [E, 4]: the alias records (thr as its uint32 bits, id, alias, 0) - what ops.csr_alias_table returns."""
    indptr, deg = _rows(indptr)
    indices = np.asarray(indices).astype(np.int64)
    E = len(indices)
    if len(deg) and deg.max(initial=0) >= MAX_ROW:
        raise ValueError("rows of 2^31 entries or more are not supported")
    N = len(deg)
    m = masses(indptr, w)
    out = np.zeros((E, 4), np.uint32)
    for v in np.nonzero(deg > 0)[0]:
        a, z = int(indptr[v]), int(indptr[v + 1])
        mv = m[a:z]
        if (mv == CAP).all():                                # every bucket full: the records are (0, id, id)
            out[a:z, 1] = indices[a:z].astype(np.uint32)
            out[a:z, 2] = indices[a:z].astype(np.uint32)
            continue
        thr, ida, al = sweep([int(x) for x in mv], indices[a:z].tolist(), N)
        out[a:z, 0] = np.asarray(thr, np.uint64).astype(np.uint32)
        out[a:z, 1] = np.asarray(ida, np.int64).astype(np.uint32)
        out[a:z, 2] = np.asarray(al, np.int64).astype(np.uint32)
    return out.view(np.int32)


def _words(seed, counter, t, j):
    t, j = np.broadcast_arrays(np.asarray(t, dtype=np.int64), np.asarray(j, dtype=np.int64))
    clo, chi = split64(counter)
    ctr = np.empty(t.shape + (4,), np.uint32)
    ctr[..., 0] = clo
    ctr[..., 1] = chi
    ctr[..., 2] = t.astype(np.uint32)
    ctr[..., 3] = (np.uint32(STREAM_ALIAS) + (j >> 1).astype(np.uint32)).astype(np.uint32)
    r = philox4x32_10(ctr, np.array(split64(seed), dtype=np.uint32))
    odd = (j & 1).astype(bool)
    return np.where(odd, r[..., 2], r[..., 0]), np.where(odd, r[..., 3], r[..., 1])


def sample(indptr, table, ids, k, seed, counter):
    """int32 [n, k]: what ops.sample_alias / one WeightedNeighborSampler call returns."""
    indptr, deg = _rows(indptr)
    N = len(deg)
    table = np.asarray(table).view(np.uint32).reshape(-1, 4)
    ids = np.asarray(ids).astype(np.int64).reshape(-1)
    n = len(ids)
    out = np.full((n, k), N, np.int32)
    if n == 0 or k == 0:
        return out
    valid = (ids >= 0) & (ids < N)
    safe = np.where(valid, ids, 0)
    d = np.where(valid, deg[safe] if N else 0, 0)
    start = np.where(valid, indptr[safe] if N else 0, 0)
    a, b = _words(seed, counter, np.arange(n)[:, None], np.arange(k)[None, :])
    live = np.broadcast_to((d > 0)[:, None], (n, k))
    bucket = mulhi32(a, np.broadcast_to(d[:, None], (n, k)).astype(np.uint32)).astype(np.int64)
    pos = np.where(live, start[:, None] + bucket, 0)
    if len(table):
        rec = table[np.minimum(pos, len(table) - 1)]
        got = np.where(b < rec[..., 0], rec[..., 1], rec[..., 2]).view(np.int32)
        out[live] = got[live]
    return out


def sample_khop(indptr, table, seeds, fanouts, seed, counter):
    """[hop 1 ids, hop 2 ids, ...] (flat int32): L single-hop calls with counters counter, counter + 1, ..."""
    outs, cur = [], np.asarray(seeds).astype(np.int32).reshape(-1)
    for h, k in enumerate(fanouts):
        cur = sample(indptr, table, cur, int(k), seed, counter + h).reshape(-1)
        outs.append(cur)
    return outs


def alias_law(table, indptr, v):
    """({id: numerator}, denominator): the exact law of one draw from row v, taking the bucket as uniform."""
    indptr, deg = _rows(indptr)
    N = len(deg)
    if not 0 <= v < N or deg[v] == 0:
        return {N: 1}, 1
    t = np.asarray(table).view(np.uint32).reshape(-1, 4)[indptr[v]:indptr[v + 1]]
    law = {}
    for thr, i, a, _ in t.tolist():
        i, a = int(np.uint32(i).view(np.int32)), int(np.uint32(a).view(np.int32))
        law[i] = law.get(i, 0) + thr
        law[a] = law.get(a, 0) + (CAP - thr)
    return {u: c for u, c in law.items() if c}, int(deg[v]) * CAP


def alias_mass_bound(n_e, d):
    """The bound on |m_j - w_j T / S| in mass units (a float; T = d 2^32)."""
    return n_e + 3 + (n_e + 8) * 2.0 ** -53 * d * CAP
