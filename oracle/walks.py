"""Oracle for the random-walk co-occurrence pairs (reference graphsage/utils.py:77-92, run_random_walks; the
`<prefix>-walks.txt` file of the unsupervised models).

Reference semantics: for every start node with G.degree(node) > 0, num_walks walks; a walk starts at curr = node and for
j = 0 .. WALK_LEN - 1 draws next = random.choice(G.neighbors(curr)), appends (node, curr) if curr != node, and moves to
next.  The last draw is never used, so a walk visits WALK_LEN - 1 nodes after the start.

RNG contract (the reference draws from Python's unseeded global `random`, which cannot be reproduced: "parity unpinned"
for the stream, pinned for the loop by tests/golden/walks.npz):
    draw s (0 <= s < L - 1) of walk w of start position i = start_offset + t is word s % 4 of
    philox4x32_10(ctr = (counter_lo, counter_hi, i, STREAM_WALK + w * ceil((L - 1) / 4) + s // 4), key = split64(seed)),
    and the step takes neighbour mulhi32(draw, deg(curr)) of curr's CSR row.
Inputs are index space: CSR indptr int64 [N+1], indices int32, starts int32.  A start outside [0, N) or without
neighbours emits nothing.  A walk that reaches a node without neighbours, or a neighbour id outside [0, N), emits it and
stops (the reference would raise IndexError; its undirected graphs never get there).  Pairs are (starts[t], visited id),
ordered by start position, then walk, then step.  Bounds: 1 <= W <= 2^20, 2 <= L <= 33.

Test infrastructure - not imported by the product.
"""
import numpy as np

from .philox import mulhi32, philox4x32_10, split64

STREAM_WALK = 0x50000000
MAX_WALKS = 1 << 20
MAX_LEN = 33


def draws(seed, counter, positions, num_walks, walk_len):
    """uint32 [len(positions), num_walks, walk_len - 1]: the draws of every walk of the given global start positions."""
    nblk = (walk_len - 1 + 3) // 4
    slo, shi = split64(seed)
    clo, chi = split64(counter)
    pos = np.asarray(positions, dtype=np.uint32)
    ctr = np.empty((len(pos), num_walks, nblk, 4), dtype=np.uint32)
    ctr[..., 0] = clo
    ctr[..., 1] = chi
    ctr[..., 2] = pos[:, None, None]
    ctr[..., 3] = (np.uint32(STREAM_WALK) + np.arange(num_walks, dtype=np.uint32)[:, None] * np.uint32(nblk)
                   + np.arange(nblk, dtype=np.uint32)[None, :])
    out = philox4x32_10(ctr, np.array([slo, shi], dtype=np.uint32))
    return out.reshape(len(pos), num_walks, nblk * 4)[..., :walk_len - 1]


class ContractChoice(object):
    """A stand-in for the `random` module of the reference's run_random_walks loop that follows the contract:
    `choice(lst)` returns lst[mulhi32(draw, len(lst))] for the loop's current (start position, walk, step), and lst[0]
    for the L-th call of a walk, whose result the loop never uses.  It tracks the loop position itself; it is told which
    start positions the loop walks from (those with G.degree(node) > 0), since the loop skips the others."""

    def __init__(self, walked_positions, num_walks, walk_len, seed, counter=0):
        self.walk_len = walk_len
        self.r = draws(seed, counter, walked_positions, num_walks, walk_len)        # [len(positions), W, L - 1]
        self.calls = 0

    def choice(self, lst):
        k, s = divmod(self.calls, self.walk_len)
        self.calls += 1
        if s == self.walk_len - 1:
            return lst[0]
        t, w = divmod(k, self.r.shape[1])
        return lst[int(mulhi32(self.r[t, w, s], len(lst)))]

    def done(self):
        """True when the loop made exactly the calls of every walk it was told about."""
        return self.calls == self.r.size // (self.walk_len - 1) * self.walk_len


def random_walks(indptr, indices, starts, num_walks, walk_len, seed, counter=0, start_offset=0):
    """int32 [P, 2] pairs of the contract above, step by step over all walks at once."""
    if not 1 <= num_walks <= MAX_WALKS or not 2 <= walk_len <= MAX_LEN:
        raise ValueError("num_walks must be in [1, %d] and walk_len in [2, %d]" % (MAX_WALKS, MAX_LEN))
    indptr = np.asarray(indptr, dtype=np.int64)
    indices = np.asarray(indices, dtype=np.int64)
    starts = np.asarray(starts, dtype=np.int64).reshape(-1)
    n_nodes = len(indptr) - 1
    n = len(starts)
    if n == 0:
        return np.zeros((0, 2), dtype=np.int32)
    start = np.repeat(starts, num_walks)                                   # walk g = t * W + w
    r = draws(seed, counter, start_offset + np.arange(n), num_walks, walk_len).reshape(n * num_walks, walk_len - 1)
    visited = np.full((n * num_walks, walk_len - 1), -1, dtype=np.int64)
    emitted = np.zeros((n * num_walks, walk_len - 1), dtype=bool)
    curr = start.copy()
    alive = (start >= 0) & (start < n_nodes)
    for j in range(walk_len - 1):
        safe = np.where(alive, curr, 0)
        row = np.where(alive, indptr[np.clip(safe, 0, n_nodes - 1)], 0) if n_nodes else np.zeros_like(safe)
        deg = np.where(alive, indptr[np.clip(safe + 1, 0, n_nodes)] - row, 0) if n_nodes else np.zeros_like(safe)
        alive &= deg > 0
        pos = mulhi32(r[:, j], np.where(alive, deg, 0).astype(np.uint32)).astype(np.int64)
        curr = np.where(alive, indices[np.where(alive, row + pos, 0)] if len(indices) else 0, curr)
        visited[:, j] = curr
        emitted[:, j] = alive & (curr != start)
        alive &= (curr >= 0) & (curr < n_nodes)
    g, j = np.nonzero(emitted)                                             # row-major: walk order, then step order
    return np.stack([start[g], visited[g, j]], axis=1).astype(np.int32)
