"""Oracle for UniformNeighborSampler (reference graphsage/neigh_samplers.py:24-29).

Reference semantics (padded mode):
    adj_lists = embedding_lookup(adj_info, ids)                     # [n, MD]   :26
    adj_lists = transpose(random_shuffle(transpose(adj_lists)))     # ONE permutation of the MD columns, shared by all rows  :27
    adj_lists = slice(adj_lists, [0,0], [-1, num_samples])          # first k columns  :28
  =>  out[i, j] = adj_info[ids[i], pi[j]],  j < k,  pi in Sym(MD) drawn once per call.

RNG contract (replaces TF's RandomShuffle stream, see oracle/philox.py):
    key = (seed_lo, seed_hi); draw number i of a call is word (i % 4) of
    philox4x32_10(ctr=(counter_lo, counter_hi, i // 4, 0), key).
    pi is built by forward Fisher-Yates:  p = [0..MD);  for i in 0..k-1:
    j = i + mulhi32(draw_i, MD - i); swap(p[i], p[j]).  Only the first k
    steps are needed for the first k entries.

CSR mode (north_star "warp-per-node random gather from a CSR adj_list"; no
reference counterpart - the reference only has the padded table) draws per node:
    draw j of node position t: word (j % 4) of
    philox4x32_10(ctr=(counter_lo, counter_hi, t, CSR_TAG + j // 4), key)
    deg == 0           -> pad_id
    deg >= k           -> Floyd's algorithm, k distinct positions
    0 < deg < k        -> replace_if_short: k iid positions mulhi32(draw_j, deg)
                          (what the padded table's choice(replace=True) rows give,
                          reference graphsage/minibatch.py:242-243); else the deg
                          neighbours in order followed by pad_id.

Test infrastructure - not imported by the product.
"""
import numpy as np

from .philox import philox4x32_10, mulhi32, split64

STREAM_PADDED = 0
STREAM_CSR = 0x40000000
STREAM_UNIGRAM = 0x20000000


def _draws(seed, counter, n_draws, c2=0, tag=STREAM_PADDED):
    """n_draws uint32 draws for one stream position (c2 may be an array -> [len(c2), n_draws])."""
    slo, shi = split64(seed)
    clo, chi = split64(counter)
    nblk = (n_draws + 3) // 4
    c2 = np.asarray(c2, dtype=np.uint32)
    ctr = np.zeros(c2.shape + (nblk, 4), dtype=np.uint32)
    ctr[..., 0] = clo
    ctr[..., 1] = chi
    ctr[..., 2] = c2[..., None]
    ctr[..., 3] = np.uint32(tag) + np.arange(nblk, dtype=np.uint32)
    out = philox4x32_10(ctr, np.array([slo, shi], dtype=np.uint32))
    return out.reshape(c2.shape + (nblk * 4,))[..., :n_draws]


def perm_prefix(seed, counter, max_deg, k):
    """First k entries of the call's column permutation pi (int32[k])."""
    assert 0 <= k <= max_deg
    p = np.arange(max_deg, dtype=np.int32)
    r = _draws(seed, counter, k)
    for i in range(k):
        j = i + int(mulhi32(r[i], max_deg - i))
        p[i], p[j] = p[j], p[i]
    return p[:k].copy()


def clamp_rows(ids, n_rows):
    """ids outside [0, n_rows) read the table's last row, the dummy row n_rows - 1 (int64)."""
    ids = np.asarray(ids).astype(np.int64)
    return np.where((ids < 0) | (ids >= n_rows), n_rows - 1, ids)


def sample_padded(adj, ids, k, seed, counter, col_perm=None):
    """out[i, j] = adj[ids[i], pi[j]]; adj int32 [N+1, MD], ids int32 [n] -> int32 [n, k].  An id outside [0, N+1)
    reads the dummy row N (clamp_rows)."""
    adj = np.asarray(adj)
    ids = clamp_rows(ids, adj.shape[0])
    pi = perm_prefix(seed, counter, adj.shape[1], k) if col_perm is None else np.asarray(col_perm)[:k]
    return adj[ids[:, None], np.asarray(pi, dtype=np.int64)[None, :]].astype(np.int32).reshape(len(ids), k)


def sample_csr(indptr, indices, ids, k, seed, counter, replace_if_short=True, pad_id=-1):
    indptr = np.asarray(indptr).astype(np.int64)
    indices = np.asarray(indices)
    ids = np.asarray(ids).astype(np.int64)
    n = len(ids)
    out = np.full((n, k), pad_id, dtype=np.int32)
    if n == 0 or k == 0:
        return out
    n_nodes = len(indptr) - 1
    valid = (ids >= 0) & (ids < n_nodes)              # ids outside [0, n_nodes) - the dummy id included - have no neighbours
    safe = np.where(valid, ids, 0)
    start = np.where(valid, indptr[safe], 0)
    deg = np.where(valid, indptr[safe + 1] - indptr[safe], 0)
    r = _draws(seed, counter, k, c2=np.arange(n, dtype=np.uint32), tag=STREAM_CSR)  # [n, k]
    # --- with replacement rows
    short = (deg > 0) & (deg < k)
    if replace_if_short:
        rows = np.nonzero(short)[0]
        if len(rows):
            pos = mulhi32(r[rows], deg[rows, None].astype(np.uint32)).astype(np.int64)
            out[rows] = indices[start[rows, None] + pos]
    else:
        for t in np.nonzero(short)[0]:
            d = int(deg[t])
            out[t, :d] = indices[start[t]:start[t] + d]
    # --- Floyd rows (deg >= k): position j draws from [0, deg-k+j]
    rows = np.nonzero(deg >= k)[0]
    if len(rows):
        d = deg[rows]
        S = np.zeros((len(rows), k), dtype=np.int64)
        for j in range(k):
            m = d - k + j
            t = mulhi32(r[rows, j], (m + 1).astype(np.uint32)).astype(np.int64)
            dup = (S[:, :j] == t[:, None]).any(axis=1) if j else np.zeros(len(rows), bool)
            S[:, j] = np.where(dup, m, t)
        out[rows] = indices[start[rows, None] + S]
    return out


def sample_unigram(degrees, num_sampled, seed, counter, distortion=0.75):
    """tf.nn.fixed_unigram_candidate_sampler(unique=False, distortion=0.75, unigrams=degrees)
    (reference graphsage/models.py:336-343): num_sampled ids with replacement, P(i) ~ deg[i]^distortion.
    Contract (TF's stream is unobtainable): draw j = word j&3 of Philox block (counter, c2=0, UNIGRAM tag + j>>2);
    u = (draw + 0.5) / 2^32 * total;  id = first index whose inclusive float64 prefix sum exceeds u."""
    cdf = np.cumsum(np.asarray(degrees, dtype=np.float64) ** distortion)
    r = _draws(seed, counter, num_sampled, c2=0, tag=STREAM_UNIGRAM).astype(np.float64)
    u = (r + 0.5) * (1.0 / 4294967296.0) * cdf[-1]
    return np.searchsorted(cdf, u, side="right").astype(np.int32)
