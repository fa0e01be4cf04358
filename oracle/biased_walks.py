"""Oracle for node2vec's second-order (p, q) random walks (Grover & Leskovec, KDD'16), drawn by rejection sampling:
the contract of gs_random_walks_biased (ops.random_walks with p, q).

Every rule of oracle/walks.py:random_walks holds (start excluded from the pairs, walk_len positions, the L-th move unused, a
start of degree 0 emits nothing, a sink or an out-of-range id ends the walk, pairs ordered by start, walk, step,
start_offset).  Only the choice of the next node changes.  From current node v, reached from t, every CSR entry x of
v's row is a candidate (duplicates count once each) of class
    return  x == t                              weight 1/p
    in      x != t and x is an entry of t's row weight 1     (the edge t -> x: node2vec's d(t, x) = 1, read directed)
    out     otherwise                           weight 1/q
quantised in float64: a = (1/p, 1, 1/q), amax = max(a), thr_c = 2^32 if a_c == amax else floor(a_c / amax * 2^32).
The chain's transition weights are exactly thr_c.  1e-4 <= p, q <= 1e4 (finite), so every thr_c >= 1.
The first move of a walk has no t: it takes entry mulhi32(word 0 of call 0, deg) and is always accepted.
Move s >= 1: attempts a = 0 .. K-1 (K = 14): candidate entry mulhi32(cand_a, deg) of v's row in its given order,
    accepted iff acc_a < thr_class(x) (as 64-bit integers).  If every attempt rejects, one exact inverse-CDF draw:
    u = w0 + 2^32 w1, target = floor(u * S / 2^64) with S = sum of thr over v's entries, and the pick is the first
    entry whose inclusive prefix sum of thr exceeds target.
An accepted candidate and the fallback have the same law, so the chain is exactly thr_x / S (up to the mulhi32
candidate pick's deg / 2^32 granularity, which the uniform walk has too).
Words: philox4x32_10(ctr = (counter_lo, counter_hi, i, STREAM_WALK_BIASED + ((w * 32 + s) << 3) + call), key = seed);
    calls 0..6 carry attempts 2 call and 2 call + 1 as (cand, acc, cand, acc), call 7's words 0, 1 are the fallback's
    u.  w < 2^20 and s < 32, so the stream spans exactly 2^28 words: [0x60000000, 0x70000000).
p == q == 1 is oracle/walks.py:random_walks, bit for bit (its own stream).

Test infrastructure - not imported by the product.
"""
import math

import numpy as np

from .philox import mulhi32, philox4x32_10, split64
from .walks import MAX_LEN, MAX_WALKS, random_walks

STREAM_WALK_BIASED = 0x60000000
ATTEMPTS = 14
PQ_MIN, PQ_MAX = 1e-4, 1e4


def check_pq(p, q):
    for name, v in (("p", p), ("q", q)):
        v = float(v)
        if not (math.isfinite(v) and PQ_MIN <= v <= PQ_MAX):
            raise ValueError("%s must be finite and in [%g, %g] (got %r)" % (name, PQ_MIN, PQ_MAX, v))


def thresholds(p, q):
    """(thr_return, thr_in, thr_out) as Python ints, float64 arithmetic exactly as the C entry does it."""
    check_pq(p, q)
    a = (1.0 / float(p), 1.0, 1.0 / float(q))
    amax = max(a)
    return tuple(1 << 32 if c == amax else int(math.floor(c / amax * 4294967296.0)) for c in a)


class _Membership(object):
    """'is x an entry of row t' for arrays of (t, x): one sorted int64 key per CSR entry, row * 2^32 + (x + 2^31)."""

    def __init__(self, indptr, indices):
        n = len(indptr) - 1
        deg = np.maximum(np.diff(indptr), 0) if n > 0 else np.zeros(0, np.int64)
        rid = np.repeat(np.arange(n, dtype=np.int64), deg)
        first = np.repeat(np.cumsum(deg) - deg, deg)
        pos = (indptr[:-1][rid] if n else rid) + np.arange(len(rid), dtype=np.int64) - first
        self.keys = np.sort(rid * (1 << 32) + indices[pos] + (1 << 31)) if len(rid) else np.zeros(0, np.int64)

    def __call__(self, t, x):
        q = np.asarray(t, np.int64) * (1 << 32) + np.asarray(x, np.int64) + (1 << 31)
        if not len(self.keys):
            return np.zeros(q.shape, bool)
        at = np.minimum(np.searchsorted(self.keys, q), len(self.keys) - 1)
        return self.keys[at] == q


def _classify(member, thr, t, x):
    """uint64 thr of each candidate x of a walk that came from t."""
    thr = np.asarray(thr, dtype=np.uint64)
    return np.where(x == t, thr[0], np.where(member(t, x), thr[1], thr[2]))


def transition_probs(indptr, indices, t, v, p, q):
    """float64 [deg(v)]: the exact law thr_x / sum(thr) of the move from v (reached from t) over v's CSR entries."""
    indptr = np.asarray(indptr, dtype=np.int64)
    indices = np.asarray(indices, dtype=np.int64)
    x = indices[indptr[v]:indptr[v + 1]]
    w = _classify(_Membership(indptr, indices), thresholds(p, q), np.full(len(x), t), x).astype(np.float64)
    return w / w.sum()


def _words(clo, chi, key, pos, word3):
    ctr = np.empty((len(pos), 4), dtype=np.uint32)
    ctr[:, 0], ctr[:, 1], ctr[:, 2], ctr[:, 3] = clo, chi, pos, word3
    return philox4x32_10(ctr, key)


def _mulhi64(a, b):
    """floor(a * b / 2^64) for uint64 arrays (exact, Python integers)."""
    return np.array([(int(x) * int(y)) >> 64 for x, y in zip(a, b)], dtype=np.uint64)


def walk_paths(indptr, indices, starts, num_walks, walk_len, p, q, seed, counter=0, start_offset=0):
    """The biased walks' paths: (visited int64 [n * W, L - 1], moved bool [n * W, L - 1], stats).  visited[g, s] is the
    node after move s of walk g = t * W + w when moved[g, s]; stats counts the moves from s >= 1 ("steps"), their
    rejection attempts ("attempts", K for a fallback) and the fallbacks ("fallbacks")."""
    if not 1 <= num_walks <= MAX_WALKS or not 2 <= walk_len <= MAX_LEN:
        raise ValueError("num_walks must be in [1, %d] and walk_len in [2, %d]" % (MAX_WALKS, MAX_LEN))
    thr = thresholds(p, q)
    indptr = np.asarray(indptr, dtype=np.int64)
    indices = np.asarray(indices, dtype=np.int64)
    starts = np.asarray(starts, dtype=np.int64).reshape(-1)
    n_nodes, n = len(indptr) - 1, len(starts)
    G = n * num_walks
    member = _Membership(indptr, indices)
    key = np.array(split64(seed), dtype=np.uint32)
    clo, chi = split64(counter)
    start = np.repeat(starts, num_walks)
    pos = (start_offset + np.repeat(np.arange(n, dtype=np.int64), num_walks)).astype(np.uint32)
    w = np.tile(np.arange(num_walks, dtype=np.int64), n)
    visited = np.full((G, walk_len - 1), -1, dtype=np.int64)
    moved = np.zeros((G, walk_len - 1), dtype=bool)
    stats = {"steps": 0, "attempts": 0, "fallbacks": 0}
    curr, prev = start.copy(), np.full(G, -1, np.int64)
    alive = (start >= 0) & (start < n_nodes)
    for s in range(walk_len - 1):
        g = np.nonzero(alive)[0]
        row = indptr[curr[g]]
        deg = indptr[curr[g] + 1] - row
        keep = deg > 0
        alive[g[~keep]] = False
        g, row, deg = g[keep], row[keep], deg[keep]
        base = (STREAM_WALK_BIASED + ((w[g] * 32 + s) << 3)).astype(np.uint32)
        nxt = np.empty(len(g), np.int64)
        if s == 0:
            r = _words(clo, chi, key, pos[g], base)
            nxt[:] = indices[row + mulhi32(r[:, 0], deg.astype(np.uint32)).astype(np.int64)]
        else:
            stats["steps"] += len(g)
            pend = np.arange(len(g))                                        # positions in g still drawing
            for call in range(ATTEMPTS // 2):
                if not len(pend):
                    break
                r = _words(clo, chi, key, pos[g[pend]], base[pend] + np.uint32(call))
                for h in (0, 1):
                    stats["attempts"] += len(pend)
                    x = indices[row[pend] + mulhi32(r[:, 2 * h], deg[pend].astype(np.uint32)).astype(np.int64)]
                    ok = r[:, 2 * h + 1].astype(np.uint64) < _classify(member, thr, prev[g[pend]], x)
                    nxt[pend[ok]] = x[ok]
                    pend, r = pend[~ok], r[~ok]
            if len(pend):
                stats["fallbacks"] += len(pend)
                r = _words(clo, chi, key, pos[g[pend]], base[pend] + np.uint32(7))
                u = r[:, 0].astype(np.uint64) | (r[:, 1].astype(np.uint64) << np.uint64(32))
                d = deg[pend]
                seg = np.repeat(np.arange(len(pend)), d)
                first = np.repeat(np.cumsum(d) - d, d)
                ent = row[pend][seg] + np.arange(len(seg), dtype=np.int64) - first
                x = indices[ent]
                wt = _classify(member, thr, prev[g[pend]][seg], x)
                incl = np.cumsum(wt)                                        # < 2^63: deg < 2^31, thr <= 2^32
                before = np.concatenate([[0], incl])[np.cumsum(d) - d].astype(np.uint64)
                local = incl - before[seg]
                total = local[np.cumsum(d) - 1]
                target = _mulhi64(u, total)
                hit = np.where(local > target[seg], np.arange(len(seg)), len(seg))
                nxt[pend] = x[np.minimum.reduceat(hit, np.cumsum(d) - d)]
        prev[g] = curr[g]
        curr[g] = nxt
        visited[g, s] = nxt
        moved[g, s] = True
        alive[g] &= (nxt >= 0) & (nxt < n_nodes)
    return visited, moved, stats


def biased_random_walks(indptr, indices, starts, num_walks, walk_len, p, q, seed, counter=0, start_offset=0,
                        stats=False):
    """int32 [P, 2] pairs of the biased walk (contract above); p == q == 1 gives random_walks' pairs.  stats=True also
    returns walk_paths' counters (all zero for p == q == 1)."""
    check_pq(p, q)
    if float(p) == 1.0 and float(q) == 1.0:
        pairs = random_walks(indptr, indices, starts, num_walks, walk_len, seed, counter, start_offset)
        return (pairs, {"steps": 0, "attempts": 0, "fallbacks": 0}) if stats else pairs
    visited, moved, st = walk_paths(indptr, indices, starts, num_walks, walk_len, p, q, seed, counter, start_offset)
    start = np.repeat(np.asarray(starts, dtype=np.int64).reshape(-1), num_walks)
    g, j = np.nonzero(moved & (visited != start[:, None]))
    pairs = np.stack([start[g], visited[g, j]], axis=1).astype(np.int32)
    return (pairs, st) if stats else pairs
