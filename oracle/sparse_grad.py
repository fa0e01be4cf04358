"""Operand-exact references for the sparse-gradient kernels: gs_embedding_grad, gs_embedding_grad_dropout and
gs_embedding_sgd (graphsage_b200/csrc/embed_grad.cu) bit for bit, and gs_skipgram_grad (csrc/skipgram.cu) exactly where
its arithmetic is a fixed fp32 chain and within derived bounds where it calls expf / log1pf.

Embedding gradient, the summation order of include/graphsage_b200.h, step by step:
  1. Number the contributions of the non-empty lists in call order (list 0 first, i ascending).  An id outside
     [0, n_rows) contributes nothing (the kernels give it the sentinel key n_rows, so it sorts last).
  2. Sort by (id, number) - a stable sort by id.
  3. Cut the sorted sequence into chunks of 32.
  4. Within a chunk each run of one id is a piece: acc = +0, then acc = fl32(acc + term) left to right, where the term
     of contribution i of list l is fl32(scale_l * grad_l[i // group_l]).
  5. With dropout sites the term is fl32(fl32(scale * g) / keep) where oracle.dropout.keep_mask(seed, call, rate,
     pos=i, F=d) keeps the element and +0 where it does not; i is the index within the list and the site is the one of
     the list's own (uncompacted) index.
  6. A run inside one chunk is the row.
  7. A run over several chunks has pieces q = 0 .. P-1.  Accumulator u of lane p (u < 4, p < 8) adds the pieces
     q = p + 8u + 32t in ascending t from +0; a lane adds its accumulators 0..3 in order; the row is lane 0 + ... + lane 7.
  8. Untouched rows are +0.
gs_embedding_sgd forms the same row sum and stores table[r] = fma32(alpha, sum, table[r]) (one rounding) for the
touched rows; every other element of the table is neither read nor written.

fma32 is fp32's fused multiply-add with one rounding.  Python 3.12 has no math.fma and a plain float64 round trip rounds
twice, so it rounds to odd in float64 first (see fma32).

Skip-gram step (gs_skipgram_grad), in the style of oracle/seq.py: the exact parts exactly, the rest teacher-forced on the
kernel's own outputs, with the bounds derived in skipgram_reference.

Test infrastructure - not imported by the product.
"""
import numpy as np

from . import dropout as _dropout
from .seq import EXPF_ULP, FLT_MIN, TINY, U, _add, _apply, _rnd

CHUNK = 32               # sorted contributions per chunk (one warp of the chunk pass)
LANES, ACCS = 8, 4       # the combine pass: piece lanes x accumulators per lane
ROWS_PER_CTA = 8         # skip-gram: one warp per pair
MAX_CTAS = 256           # skip-gram: the fixed grid cap
# CUDA C++ Programming Guide, "Mathematical Functions", single precision (CUDA 12): log1pf has a maximum error of 1 ulp.
LOG1PF_ULP = 1
# criterion (b)-style RMS statistic: sqrt(mean((max(|out - ref| - R, 0) / S2)^2)) with R the operand allowance of each
# output and S2 = sqrt(m + 1) u S1 for a chain of m roundings over terms of absolute sum S1 - the scale at which errors
# that round either way add up, against the worst case's (m + 1) u S1.  A kernel whose roundings lean one way (a
# truncating add, a dropped term's worth of drift) reaches about sqrt(m) / 2 of it on long chains.
RMS_BOUND = 1.0


def fma32(a, b, c):
    """fp32 fma(a, b, c) with one rounding, elementwise (numpy broadcasting).  a b is exact in float64 (48 significant
    bits); s = fl64(a b + c) and its exact error come from TwoSum; s is rounded to odd (a non-zero error and an even last
    significand bit step s one ulp toward the error) and then cast to float32.  Rounding to odd at 53 >= 24 + 2 bits makes
    that cast the correctly rounded result, subnormal results included."""
    a, b, c = np.broadcast_arrays(*(np.asarray(x, np.float32).astype(np.float64) for x in (a, b, c)))
    with np.errstate(invalid="ignore", over="ignore"):
        p = a * b
        s = p + c
        bb = s - p
        err = (p - (s - bb)) + (c - bb)
        even = (np.ascontiguousarray(s).view(np.uint64) & np.uint64(1)) == 0
        fix = np.isfinite(s) & (err != 0) & even
        s = np.where(fix, np.nextafter(s, np.where(err > 0, np.inf, -np.inf)), s)
        return s.astype(np.float32)


# ---------------------------------------------------------------------------------------------------- embedding grad
def sorted_terms(lists, n_rows, d, sites=None):
    """Steps 1, 2 and 5: (keys [T] int64 with n_rows for ids outside the table, terms [T, d] float32) in sorted order.
    lists: (ids, grad [>= ceil(n / group), >= d], group, scale) numpy; sites: one (seed, call, rate) per list or None."""
    keys, terms = [], []
    for l, (ids, grad, group, scale) in enumerate(lists):
        ids = np.asarray(ids, np.int64).reshape(-1)
        if ids.size == 0:
            continue
        i = np.arange(ids.size)
        ok = (ids >= 0) & (ids < n_rows)
        g = np.asarray(grad, np.float32)[i // int(group), :d]
        with np.errstate(invalid="ignore", over="ignore"):
            t = np.float32(scale) * g
            if sites is not None:
                seed, call, rate = sites[l][:3]
                t = np.where(_dropout.keep_mask(seed, call, rate, i, d), t / _dropout.keep_prob(rate), np.float32(0))
        keys.append(np.where(ok, ids, n_rows))
        terms.append(np.where(ok[:, None], t, np.float32(0)).astype(np.float32))
    if not keys:
        return np.zeros(0, np.int64), np.zeros((0, d), np.float32)
    keys, terms = np.concatenate(keys), np.concatenate(terms)
    order = np.argsort(keys, kind="stable")
    return keys[order], terms[order]


def chunk_sums(keys, terms):
    """Step 4: the running fp32 sum of every piece at every sorted position, [T, d] (a piece's value sits at its last
    position).  One masked vector add per chunk position over a [chunks, 32, d] array."""
    T, d = terms.shape
    nch = -(-T // CHUNK)
    K = np.full(nch * CHUNK, -1, np.int64)
    K[:T] = keys
    X = np.zeros((nch * CHUNK, d), np.float32)
    X[:T] = terms
    K, X = K.reshape(nch, CHUNK), X.reshape(nch, CHUNK, d)
    start = np.ones((nch, CHUNK), bool)
    start[:, 1:] = K[:, 1:] != K[:, :-1]
    run = np.empty_like(X)
    acc = np.zeros((nch, d), np.float32)
    with np.errstate(invalid="ignore", over="ignore"):
        for i in range(CHUNK):
            acc = np.where(start[:, i, None], np.float32(0), acc) + X[:, i]
            run[:, i] = acc
    return run.reshape(nch * CHUNK, d)[:T]


def combine_pieces(pieces):
    """Step 7 for one run's pieces [P, d]: piece q to accumulator (q // 8) % 4 of lane q % 8, fp32."""
    P, d = pieces.shape
    pad = np.zeros((-(-P // (LANES * ACCS)) * LANES * ACCS, d), np.float32)
    pad[:P] = pieces
    pad = pad.reshape(-1, ACCS, LANES, d)                      # [t, u, p]: q = 32 t + 8 u + p
    a = np.zeros((ACCS, LANES, d), np.float32)
    with np.errstate(invalid="ignore", over="ignore"):
        for t in range(pad.shape[0]):
            a = a + pad[t]
        lane = a[0]
        for u in range(1, ACCS):
            lane = lane + a[u]
        row = lane[0]
        for p in range(1, LANES):
            row = row + lane[p]
    return row


def row_sums(keys, terms, n_rows):
    """Steps 3, 4, 6 and 7 on sorted (keys, terms): (touched row ids, their sums [rows, d]) in ascending id."""
    T, d = terms.shape
    if T == 0:
        return np.zeros(0, np.int64), np.zeros((0, d), np.float32)
    run = chunk_sums(keys, terms)
    b = np.flatnonzero(np.r_[keys[1:] != keys[:-1], True]) + 1      # run ends (exclusive)
    a = np.r_[0, b[:-1]]
    live = keys[a] < n_rows
    a, b = a[live], b[live]
    ids = keys[a]
    sums = run[b - 1].copy()
    ja, jb = a // CHUNK, (b - 1) // CHUNK
    for r in np.flatnonzero(ja != jb):
        ends = np.r_[np.arange(ja[r], jb[r]) * CHUNK + CHUNK - 1, b[r] - 1]
        sums[r] = combine_pieces(run[ends])
    return ids, sums


def embedding_grad_reference(lists, n_rows, d, sites=None):
    """gs_embedding_grad (sites None) / gs_embedding_grad_dropout, bit for bit: float32 [n_rows, d]."""
    ids, sums = row_sums(*sorted_terms(lists, n_rows, d, sites), n_rows)
    out = np.zeros((n_rows, d), np.float32)
    out[ids] = sums
    return out


def embedding_sgd_reference(table, lists, alpha, d=None):
    """gs_embedding_sgd, bit for bit: a copy of table (float32 [n_rows, >= d]) with table[r, :d] = fma32(alpha, sum_r,
    table[r, :d]) for the touched rows; every other element keeps its bits (NaN payloads included)."""
    out = np.array(table, np.float32, copy=True)
    d = out.shape[1] if d is None else d
    ids, sums = row_sums(*sorted_terms(lists, out.shape[0], d), out.shape[0])
    if ids.size:
        out[ids, :d] = fma32(np.float32(alpha), sums, out[ids, :d])
    return out


# ---------------------------------------------------------------------------------------------------- skip-gram
def n_ctas(B):
    return min(-(-B // ROWS_PER_CTA), MAX_CTAS)


def butterfly(v):
    """The xor butterfly of a warp: v_l = fl32(v_l + v_{l ^ o}) for o = 16, 8, 4, 2, 1 over the last axis (32 lanes);
    fp32 addition commutes, so every lane ends with the same bits.  Returns lane 0."""
    idx = np.arange(32)
    with np.errstate(invalid="ignore", over="ignore"):
        for o in (16, 8, 4, 2, 1):
            v = v + v[..., idx ^ o]
    return v[..., 0]


def lane_dot(x, y):
    """The kernel's dot product of x [..., d] and y [..., d] (broadcast): lane l holds s = +0 and s = fma32(x_q, y_q, s)
    for q = l, l + 32, ...; then the butterfly."""
    d = x.shape[-1]
    s = np.zeros(np.broadcast_shapes(x.shape[:-1], y.shape[:-1]) + (32,), np.float32)
    for k0 in range(0, d, 32):
        w = min(32, d - k0)
        s[..., :w] = fma32(x[..., k0:k0 + w], y[..., k0:k0 + w], s[..., :w])
    return butterfly(s)


def lookup(table, ids, cols):
    """table[ids, :cols] as float32, with a zero row for ids outside [0, n_rows)."""
    ids = np.asarray(ids, np.int64).reshape(-1)
    ok = (ids >= 0) & (ids < table.shape[0])
    rows = np.asarray(table, np.float32)[np.where(ok, ids, 0), :cols]
    return np.where(ok[:, None], rows, np.float32(0))


def skipgram_operands(target, context, d, batch1, batch2, neg):
    """(t [B, d], c [B, d], b [B], n [S, d], nb [S]) float32, zero rows and biases for ids outside the tables."""
    c, n = lookup(context, batch2, d + 1), lookup(context, neg, d + 1)
    return lookup(target, batch1, d), c[:, :d], c[:, d], n[:, :d], n[:, d]


def skipgram_affinities(t, c, n, block=64):
    """aff [B] and neg_aff [B, S] as the kernel forms them, bit for bit."""
    aff = lane_dot(t, c)
    neg_aff = np.empty((t.shape[0], n.shape[0]), np.float32)
    for i0 in range(0, t.shape[0], block):
        neg_aff[i0:i0 + block] = lane_dot(t[i0:i0 + block, None, :], n[None, :, :])
    return aff, neg_aff


def _softplus(x):
    """softplus(x) = fmaxf(x, 0) + log1pf(expf(-|x|)) on an exact fp32 operand: (float64 value, bound).  expf: 2 ulp
    (<= 2 EXPF_ULP u relative) plus FLT_MIN for a result it flushes; log1p moves by at most that much (slope <= 1);
    log1pf: LOG1PF_ULP ulp; then one rounding of the add."""
    y = np.exp(-np.abs(x))
    ey = 2 * EXPF_ULP * U * y + FLT_MIN
    L = np.log1p(y)
    eL = ey + 2 * LOG1PF_ULP * U * (L + ey) + TINY
    return _add((np.maximum(x, 0.0), 0.0), (L, eL))


def skipgram_reference(target, context, d, batch1, batch2, neg, aff, neg_aff, gc_pos):
    """Reference of one gs_skipgram_grad call, teacher-forced on the kernel's own aff [B], neg_aff [B, S] and g (its
    gc_pos[:, d]).  Returns {"aff", "neg_aff", "gc_pos_rows": exact float32 arrays} and, for the bounded outputs
    "g" [B], "gt" [B, d], "gc_neg" [S, d + 1] and "loss" [1], (ref, bound, s2, r) float64 tuples (check_bounded).

    Exact parts (the kernel's fp32 chains on exactly these operands):
      aff_i = lane_dot(t_i, c_i), neg_aff_ij = lane_dot(t_i, n_j): per-lane fma32 chains from +0, then the butterfly.
      gc_pos[i, :d] = fl32(g_i t_i) with the kernel's own g_i.
    Bounded parts, on the kernel's exact logits x_i = fl32(aff_i + b_i) and x_ij = fl32(neg_aff_ij + nb_j) (u = 2^-24):
      sigma(x) = 1 / (1 + expf(-x)): oracle.seq's rule - SIGMOID_REL relative (expf 2 ulp, the add, the division, 1 u
          spare) plus FLT_MIN, and its slope rule for an operand error (here 0: x is exact).
      g_i = fl32(fl32(sigma(x_i) - 1) / B), h_ij = fl32(sigma(x_ij) / B): one rounding per operation (seq._add, _rnd);
          fp32(B) is exact for B < 2^24.  Call their bounds e_g, e_h and write G = |g| + e_g, H = |h| + e_h.
      gt[i, q] = fl32(g_i c_iq), then fma32(h_ij, n_jq, .) for j = 0 .. S-1: S + 1 roundings, so
          |gt - ref| <= e_g |c_iq| + sum_j e_h,ij |n_jq| + (S + 2) u (G |c_iq| + sum_j H_ij |n_jq|) + (S + 1) 2^-149
          (gamma_{S+1} <= (S + 2) u; each rounding that underflows adds at most 2^-149).
      gc_neg[j, q] = sum_i h_ij t_iq (t_id = 1 for the bias column): CTA k chains fma32 over the rows of its groups
          k, k + grid, ... in group order from +0 (at most m_1 = 8 ceil(ceil(B / 8) / grid) roundings), then the grid
          partials are added in CTA order (grid - 1 roundings).  With m = m_1 + grid - 1:
          |gc_neg - ref| <= sum_i e_h,ij |t_iq| + (m + 1) u sum_i H_ij |t_iq| + m 2^-149.
      loss = fl32(L / B), L the fp32 sum of the B S + B softplus terms: per row softplus(-x_i) then + softplus(x_ij)
          in j order (S roundings), lane l adds rows l, l + 32, ... from +0 (ceil(B / 32) roundings), then the
          butterfly (5).  Each softplus is known within e_sp (_softplus), so with m = S + ceil(B / 32) + 5:
          |L - sum sp| <= sum e_sp + (m + 1) u sum (|sp| + e_sp) + (m + 1) 2^-149, then the division's rounding (_rnd).
    RMS statistic (check_bounded): R is each output's operand allowance (the e_g, e_h and e_sp terms, and the final
    division's rounding for the loss), S2 = sqrt(m + 1) u S1 for its chain of m roundings (m = S + 1 for gt); the
    statistic must stay below RMS_BOUND, so a kernel cannot sit consistently near its worst-case bound.  For g the
    statistic is 0 by construction (R is its whole bound)."""
    t, c, b, n, nb = skipgram_operands(target, context, d, batch1, batch2, neg)
    B, S = t.shape[0], n.shape[0]
    aff, neg_aff = np.asarray(aff, np.float32), np.asarray(neg_aff, np.float32)
    g_k = np.asarray(gc_pos, np.float32)[:, d]
    ex_aff, ex_neg = skipgram_affinities(t, c, n)
    out = {"aff": ex_aff, "neg_aff": ex_neg, "gc_pos_rows": (g_k[:, None] * t).astype(np.float32)}
    with np.errstate(over="ignore"):
        x = (aff + b).astype(np.float64)
        xn = (neg_aff + nb[None, :]).astype(np.float64)
    sg = _apply("sigmoid", (x, np.zeros_like(x)))
    sn = _apply("sigmoid", (xn, np.zeros_like(xn)))
    gm = _add(sg, (-1.0, 0.0))
    g, eg = _rnd(gm[0] / B, gm[1] / B)
    h, eh = _rnd(sn[0] / B, sn[1] / B)
    G, H = np.abs(g) + eg, np.abs(h) + eh
    t64, c64, n64 = t.astype(np.float64), c.astype(np.float64), n.astype(np.float64)
    # gt
    ref = g[:, None] * c64 + h @ n64
    R = eg[:, None] * np.abs(c64) + eh @ np.abs(n64)
    S1 = G[:, None] * np.abs(c64) + H @ np.abs(n64)
    out["gt"] = (ref, R + (S + 2) * U * S1 + (S + 1) * TINY, np.sqrt(S + 2) * U * S1, R)
    out["g"] = (g, eg, np.abs(g), eg)
    # gc_neg (column d: t = 1)
    t1 = np.concatenate([t64, np.ones((B, 1))], axis=1)
    grid = n_ctas(B)
    groups = -(-B // ROWS_PER_CTA)
    m = ROWS_PER_CTA * -(-groups // grid) + grid - 1
    ref = h.T @ t1
    R = eh.T @ np.abs(t1)
    S1 = H.T @ np.abs(t1)
    out["gc_neg"] = (ref, R + (m + 1) * U * S1 + m * TINY, np.sqrt(m + 1) * U * S1, R)
    # loss
    sp, esp = _softplus(-x)
    spn, espn = _softplus(xn)
    total = sp.sum() + spn.sum()
    e_op = esp.sum() + espn.sum()
    m = S + -(-B // 32) + 5
    e_sum = e_op + (m + 1) * U * (np.abs(sp).sum() + np.abs(spn).sum() + e_op) + (m + 1) * TINY
    ref, bound = _rnd(total / B, e_sum / B)
    s2 = np.sqrt(m + 1) * U * (np.abs(sp).sum() + np.abs(spn).sum()) / B
    out["loss"] = tuple(np.array([v], np.float64) for v in (ref, bound, s2, e_op / B + U * abs(ref) + TINY))
    return out


def errors(out, ref, bound, s2, r):
    """(worst, rms): worst = max |out - ref| / bound (a NaN or inf output is inf), rms = the module's RMS statistic."""
    out = np.asarray(out, np.float64)
    err = np.where(np.isfinite(out), np.abs(out - ref), np.inf)
    if err.size == 0:
        return 0.0, 0.0
    worst = float(np.divide(err, bound, out=np.where(err > 0, np.inf, 0.0), where=bound > 0).max())
    acc = np.maximum(err - r, 0.0)
    rel = np.divide(acc, s2, out=np.where(acc > 0, np.inf, 0.0), where=s2 > 0)
    return worst, float(np.sqrt(np.mean(rel * rel)))


def check_bounded(out, ref, bound, s2, r, rms_bound=RMS_BOUND):
    """(ok, worst, rms): |out - ref| <= bound everywhere and the RMS statistic <= rms_bound."""
    worst, rms = errors(out, ref, bound, s2, r)
    return worst <= 1.0 and rms <= rms_bound, worst, rms


BOUNDED = ("g", "gt", "gc_neg", "loss")


def check_skipgram(target, context, d, batch1, batch2, neg, got):
    """Every check of one gs_skipgram_grad call.  got: numpy loss (scalar), aff [B], neg_aff [B, S], gt [B, d],
    gc_pos [B, d + 1], gc_neg [S, d + 1].  Returns (failures: list of output names, {name: (worst, rms)})."""
    ref = skipgram_reference(target, context, d, batch1, batch2, neg, got["aff"], got["neg_aff"], got["gc_pos"])
    fails = []
    for name, have in (("aff", got["aff"]), ("neg_aff", got["neg_aff"]), ("gc_pos_rows", got["gc_pos"][:, :d])):
        a, e = np.asarray(have, np.float32), ref[name]
        if not (a.shape == e.shape and np.array_equal(a.view(np.uint32), e.view(np.uint32))):
            fails.append(name)
    stats = {}
    have = {"g": np.asarray(got["gc_pos"])[:, d], "gt": got["gt"], "gc_neg": got["gc_neg"],
            "loss": np.reshape(np.asarray(got["loss"], np.float64), (1,))}
    for name in BOUNDED:
        ok, worst, rms = check_bounded(have[name], *ref[name])
        stats[name] = (worst, rms)
        if not ok:
            fails.append(name)
    return fails, stats
