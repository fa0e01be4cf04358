"""CPU: oracle/sparse_grad.py - the contract tests/test_zz_gpu_sparse_grad.py holds the sparse-gradient kernels to - and
the evidence that its checks have teeth.  fma32 agrees with exact rational arithmetic; the references agree with the
fp64 semantics the older tests check; a numpy emulation of the kernels (the chunk pass with its partial slots, the
combine pass, the skip-gram rows and combine kernels) passes every check at the GPU file's shapes; and each mutant below
(a subtly wrong kernel) fails a check the GPU file applies, at one of its shapes."""
from fractions import Fraction

import numpy as np
import pytest
import torch

from oracle import dropout as od
from oracle import node2vec as on2v
from oracle import sparse_grad as sg
from test_zz_gpu_identity import _check_grad
from test_zz_gpu_sparse_grad import (EMBED_D, SG_CASES, edge_layout, embed_case, embed_sites, reddit_case, sg_case,
                                     sgd_case)

EMBED_MUTANTS = {
    "ascending_q": "grad",          # the pieces of a crossing run added in plain ascending q
    "first_slot_2j": "grad",        # a crossing run's first piece read from slot 2j although it began mid-chunk
    "fma_chunk": "grad",            # acc = fma(scale, g, acc): the chunk pass contracted
    "sgd_two_roundings": "sgd",     # table + fl32(alpha * sum) instead of one fma
    "unstable_sort": "grad",        # the contributions of one id in reverse number order
    "grad_row_mod": "grad",         # contribution i reads grad row i % group
    "drop_pos_global": "dropout",   # the dropout position is the global contribution number, not the index in the list
    "site_compacted": "dropout",    # the site of the compacted list index: an empty list shifts the later lists' sites
    "tile2_skipped": "grad",        # the second 128-column tile of the chunk pass skipped
}
SG_MUTANTS = [
    "bias_in_aff",          # the bias included in aff
    "sequential_lanes",     # the dot products' lanes added in order instead of by the butterfly
    "h_not_divided",        # h not divided by B
    "cta_overwrite",        # a CTA's second pair group overwrites its gc_neg partial instead of adding to it
    "gt_without_gc",        # gt without the g c term
    "nb_from_positive",     # the negatives' logits biased with the positive row's b_i instead of nb_j
]


def _f32(x):
    return np.float32(x)


# ---------------------------------------------------------------------------------------------------- fma32
def _round_f32(q):
    """The float32 nearest to the rational q, ties to even (subnormals and overflow included)."""
    x = np.float32(float(q))
    best = None
    for c in (np.nextafter(x, np.float32(-np.inf)), x, np.nextafter(x, np.float32(np.inf))):
        if not np.isfinite(c):
            continue
        dist = abs(Fraction(float(c)) - q)
        key = (dist, int(np.array(c, np.float32).view(np.uint32)) & 1)
        if best is None or key < best[0]:
            best = (key, c)
    return best[1]


def _fma_inputs():
    rs = np.random.RandomState(0)
    a = (rs.randn(3000) * 2.0 ** rs.randint(-60, 60, 3000)).astype(np.float32)
    b = (rs.randn(3000) * 2.0 ** rs.randint(-60, 60, 3000)).astype(np.float32)
    c = (rs.randn(3000) * 2.0 ** rs.randint(-60, 60, 3000)).astype(np.float32)
    cases = list(zip(a, b, c))
    one, eps = _f32(1), _f32(2.0 ** -23)
    cases += [
        (one + eps, one + eps, _f32(-1)),                            # a b = 1 + 2^-22 + 2^-46: the tail decides
        (one + eps, one - eps, _f32(0)),                            # 1 - 2^-46: just below 1
        (_f32(1.5), _f32(1 + 2 ** -23), _f32(2 ** -25)),             # halfway cases shifted by a tiny c
        (_f32(1 + 2 ** -12), _f32(1 + 2 ** -12), _f32(-(1 + 2 ** -11))),   # exact cancellation to 2^-24
        (_f32(3), _f32(1 / 3), _f32(-1)),                            # cancellation of a rounded third
        (_f32(2 ** -75), _f32(2 ** -75), _f32(0)),                   # subnormal product
        (_f32(1.5 * 2 ** -75), _f32(2 ** -75), _f32(-(2 ** -149))),  # subnormal result, halfway
        (_f32(2 ** -100), _f32(2 ** -49), _f32(2 ** -149)),          # 2^-149 + 2^-149
        (_f32(-0.0), _f32(5), _f32(0.0)), (_f32(-2), _f32(0), _f32(-0.0)), (_f32(0), _f32(3), _f32(-0.0)),
        (_f32(3.4e38), _f32(1), _f32(-3.4e38)),
    ]
    # a b = 1 + 2^-11 + 2^-24: halfway between two floats; c = +-2^-70 decides, c = 0 ties to even
    for s in (1, -1):
        cases.append((_f32(1 + 2 ** -12), _f32(1 + 2 ** -12), _f32(s * 2 ** -70)))
        cases.append((_f32(s * (1 + 2 ** -12)), _f32(1 + 2 ** -12), _f32(0)))
    return cases


def test_fma32_is_exact_rational_fma():
    cases = _fma_inputs()
    a, b, c = (np.array(x, np.float32) for x in zip(*cases))
    got = sg.fma32(a, b, c)
    for i, (x, y, z) in enumerate(cases):
        q = Fraction(float(x)) * Fraction(float(y)) + Fraction(float(z))
        want = _round_f32(q)
        if q == 0:                                                  # exact zero: the IEEE sign rule
            want = np.float32(x) * np.float32(y) + np.float32(z)
        assert np.array(got[i]).view(np.uint32) == np.array(want, np.float32).view(np.uint32), (x, y, z, got[i], want)
    # a float64 round trip rounds twice and gets at least one of these wrong: the test above can tell
    twice = (a.astype(np.float64) * b + c).astype(np.float32)
    assert not np.array_equal(twice.view(np.uint32), got.view(np.uint32))


# ---------------------------------------------------------------------------------------------------- the oracle
def _torch_lists(lists):
    return [(torch.from_numpy(ids), torch.from_numpy(g), group, scale) for ids, g, group, scale in lists]


@pytest.mark.parametrize("d", [1, 33, 129])
def test_embedding_reference_is_the_fp64_sum(d):
    """Against test_zz_gpu_identity's fp64 index_add_ criterion (1e-5 per row), on the GPU file's lists with the
    subnormal gradients flushed: the fp32 rounding of a subnormal term is not small relative to itself."""
    n_rows, lists = embed_case(d)
    lists = [(ids, np.where(np.abs(g) < 2.0 ** -126, np.float32(0), g), group, scale) for ids, g, group, scale in lists]
    got = sg.embedding_grad_reference(lists, n_rows, d)
    _check_grad(torch.from_numpy(got), _torch_lists(lists), n_rows, d)
    sites = embed_sites(lists)
    masked = sg.embedding_grad_reference(lists, n_rows, d, sites)
    dropped = []
    for l, (ids, g, group, scale) in enumerate(lists):
        n = ids.size
        x = np.repeat(g[:max(-(-n // group), 1), :d], group, axis=0)[:n]
        dropped.append((ids, od.apply(x, *sites[l], pos=np.arange(n)) if n else g, 1, scale))
    _check_grad(torch.from_numpy(masked), _torch_lists(dropped), n_rows, d)
    zero = [(s, c, 0.0) for s, c, _ in sites]
    assert np.array_equal(sg.embedding_grad_reference(lists, n_rows, d, zero).view(np.uint32), got.view(np.uint32))


def test_edge_layout_lands_on_chunk_edges():
    layout, n = edge_layout()
    starts = np.flatnonzero(np.r_[True, layout[1:] != layout[:-1]])
    lengths = np.diff(np.r_[starts, layout.size])
    seen = {(int(L), int(s % 32)) for s, L in zip(starts, lengths) if L > 1}
    assert {(L, r) for L in (31, 32, 33, 64) for r in (0, 1, 31)} <= seen
    pieces = {int((s + L - 1) // 32 - s // 32 + 1) for s, L in zip(starts, lengths) if s % 32 == 5 and L > 1}
    assert {2, 8, 9, 32, 33} <= pieces


def test_sgd_reference_is_the_fp64_update():
    table, lists = sgd_case(51)
    d, lr = 51, 0.05
    got = sg.embedding_sgd_reference(table, lists, _f32(-lr), d)
    want = table[:, :d].astype(np.float64)
    for ids, g, _, scale in lists:
        ok = (ids >= 0) & (ids < table.shape[0])
        np.add.at(want, ids[ok].astype(np.int64), -lr * scale * g[:ids.size, :d][ok].astype(np.float64))
    fin = np.isfinite(want)
    assert np.abs(got[:, :d][fin] - want[fin]).max() <= 1e-5 * max(1.0, np.abs(want[fin]).max())
    untouched = ~np.isfinite(table[:, 0])
    assert got[untouched].tobytes() == table[untouched].tobytes() and got[:, d:].tobytes() == table[:, d:].tobytes()


def test_skipgram_reference_is_the_fp64_step():
    B, S, d = 37, 20, 50
    T, C, b1, b2, neg = sg_case(B, S, d)
    t, c, b, n, nb = sg.skipgram_operands(T, C, d, b1, b2, neg)
    em = emulate_skipgram(T, C, d, b1, b2, neg)
    ref = sg.skipgram_reference(T, C, d, b1, b2, neg, em["aff"], em["neg_aff"], em["gc_pos"])
    # the fp64 semantics of oracle.node2vec on the looked-up rows (zero rows for ids outside the tables)
    Cc, bb = np.concatenate([c, n]), np.concatenate([b, nb])
    ids = (np.arange(B), np.arange(B), B + np.arange(S))
    loss, aff, neg_aff = on2v.skipgram_forward(t, Cc, bb, *ids)
    gr = on2v.skipgram_grads(t, Cc, bb, *ids)
    assert np.allclose(ref["aff"], aff, rtol=1e-4, atol=1e-5) and np.allclose(ref["neg_aff"], neg_aff, rtol=1e-4, atol=1e-5)
    assert abs(ref["loss"][0][0] - loss) <= 2e-5 * abs(loss)
    for mine, theirs in ((ref["gt"][0], gr["gt"]), (ref["g"][0], gr["gb_pos"]), (ref["gc_neg"][0][:, :d], gr["gc_neg"]),
                         (ref["gc_neg"][0][:, d], gr["gb_neg"])):
        assert np.abs(mine - theirs).max() <= 1e-5 * np.abs(theirs).max() + 1e-9
    assert np.allclose(ref["gc_pos_rows"], gr["gc_pos"], rtol=1e-5, atol=1e-9 * np.abs(gr["gc_pos"]).max())


# ---------------------------------------------------------------------------------------------------- kernel emulation
def emulate_embed(lists, n_rows, d, sites=None, mutant=None, table=None, alpha=None):
    """embed_keys_kernel + the stable radix sort + embed_chunk_kernel + embed_combine_kernel in numpy, with the
    partial slots in a NaN workspace.  table / alpha: gs_embedding_sgd (in place on a copy of table)."""
    keys, nums, rows, scales, terms = [], [], [], [], []
    off = count = 0
    for l, (ids, grad, group, scale) in enumerate(lists):
        ids = np.asarray(ids, np.int64)
        if ids.size == 0:
            continue
        i = np.arange(ids.size)
        r = (i % group) if mutant == "grad_row_mod" else i // group
        g = grad[r, :d]
        t = _f32(scale) * g
        if sites is not None:
            seed, call, rate = sites[count if mutant == "site_compacted" else l]
            pos = off + i if mutant == "drop_pos_global" else i
            t = np.where(od.keep_mask(seed, call, rate, pos, d), t / od.keep_prob(rate), _f32(0))
        ok = (ids >= 0) & (ids < n_rows)
        keys.append(np.where(ok, ids, n_rows))
        nums.append(off + i)
        rows.append(np.where(ok[:, None], g, _f32(0)))
        scales.append(np.full(ids.size, scale, np.float32))
        terms.append(np.where(ok[:, None], t, _f32(0)).astype(np.float32))
        off += ids.size
        count += 1
    out = np.zeros((n_rows, d), np.float32) if table is None else np.array(table, np.float32, copy=True)
    if off == 0:
        return out
    keys, nums = np.concatenate(keys), np.concatenate(nums)
    order = np.lexsort((-nums, keys)) if mutant == "unstable_sort" else np.argsort(keys, kind="stable")
    keys, rows, scales, terms = keys[order], np.concatenate(rows)[order], np.concatenate(scales)[order], \
        np.concatenate(terms)[order]
    total = keys.size
    nch = -(-total // 32)
    dcols = min(d, 128) if mutant == "tile2_skipped" else d
    K = np.full(nch * 32, n_rows, np.int64)
    K[:total] = keys
    K = K.reshape(nch, 32)
    pad = lambda a: np.concatenate([a, np.zeros((nch * 32 - total,) + a.shape[1:], a.dtype)]).reshape((nch, 32) + a.shape[1:])  # noqa
    X, G, SC = pad(terms[:, :dcols]), pad(rows[:, :dcols]), pad(scales)
    cnt = np.minimum(32, total - np.arange(nch) * 32)
    key_before = np.r_[-1, keys[np.arange(1, nch) * 32 - 1]] if nch > 1 else np.array([-1])
    after_idx = np.arange(nch) * 32 + cnt
    key_after = np.where(after_idx < total, keys[np.minimum(after_idx, total - 1)], -1)
    partial = np.full((2 * nch, d), np.nan, np.float32)
    acc = np.zeros((nch, dcols), np.float32)
    piece_start = np.zeros(nch, np.int64)
    with np.errstate(invalid="ignore", over="ignore"):
        for i in range(32):
            if mutant == "fma_chunk":
                acc = sg.fma32(SC[:, i, None], G[:, i], acc)
            else:
                acc = acc + X[:, i]
            nxt = K[:, i + 1] if i < 31 else np.full(nch, -2)
            end = (i < cnt) & ((i == cnt - 1) | (nxt != K[:, i]))
            js = np.flatnonzero(end & (K[:, i] < n_rows))
            key = K[js, i]
            before = (piece_start[js] == 0) & (key_before[js] == key)
            after = (i == cnt[js] - 1) & (key_after[js] == key)
            whole = ~before & ~after
            w, kw = js[whole], key[whole]
            if table is None:
                out[kw, :dcols] = acc[w]
            elif mutant == "sgd_two_roundings":
                out[kw, :dcols] = out[kw, :dcols] + _f32(alpha) * acc[w]
            else:
                out[kw, :dcols] = sg.fma32(_f32(alpha), acc[w], out[kw, :dcols])
            slot = 2 * js[~whole] + (piece_start[js[~whole]] != 0)
            partial[slot, :dcols] = acc[js[~whole]]
            acc[end] = 0
            piece_start[end] = i + 1
        for j in range(nch):
            s, e = 32 * j, 32 * j + 32
            if e >= total or keys[e - 1] >= n_rows or keys[e] != keys[e - 1] or (s > 0 and keys[s - 1] == keys[e - 1]):
                continue
            X_ = keys[e - 1]
            run_end = np.searchsorted(keys, X_, side="right")
            npieces = (run_end - 1) // 32 - j + 1
            first = 2 * j if keys[s] == X_ or mutant == "first_slot_2j" else 2 * j + 1
            pieces = partial[[first] + [2 * (j + q) for q in range(1, npieces)]]
            if mutant == "ascending_q":
                r = np.zeros(d, np.float32)
                for p in pieces:
                    r = r + p
            else:
                r = sg.combine_pieces(pieces)
            if table is None:
                out[X_] = r
            elif mutant == "sgd_two_roundings":
                out[X_, :d] = out[X_, :d] + _f32(alpha) * r
            else:
                out[X_, :d] = sg.fma32(_f32(alpha), r, out[X_, :d])
    return out


def emulate_skipgram(T, C, d, b1, b2, neg, mutant=None):
    """skipgram_rows_kernel + skipgram_combine_kernel in numpy (sigma and softplus in float64, rounded once)."""
    t, c, b, n, nb = sg.skipgram_operands(T, C, d, b1, b2, neg)
    B, S = t.shape[0], n.shape[0]
    if mutant == "sequential_lanes":
        def dot(x, y):
            s = np.zeros(np.broadcast_shapes(x.shape[:-1], y.shape[:-1]) + (32,), np.float32)
            for k0 in range(0, d, 32):
                w = min(32, d - k0)
                s[..., :w] = sg.fma32(x[..., k0:k0 + w], y[..., k0:k0 + w], s[..., :w])
            r = s[..., 0]
            for l in range(1, 32):
                r = r + s[..., l]
            return r
        aff, neg_aff = dot(t, c), dot(t[:, None, :], n[None, :, :])
    else:
        aff, neg_aff = sg.skipgram_affinities(t, c, n)
    x = aff + b
    if mutant == "bias_in_aff":
        aff = x
    xn = neg_aff + (b[:, None] if mutant == "nb_from_positive" else nb[None, :])
    sig = lambda v: (1.0 / (1.0 + np.exp(-v.astype(np.float64)))).astype(np.float32)    # noqa: E731
    fB = _f32(B)
    g = (sig(x) - _f32(1)) / fB
    h = sig(xn) if mutant == "h_not_divided" else sig(xn) / fB
    gt = np.zeros((B, d), np.float32) if mutant == "gt_without_gc" else g[:, None] * c
    for j in range(S):
        gt = sg.fma32(h[:, j, None], n[None, j], gt)
    gc_pos = np.concatenate([g[:, None] * t, g[:, None]], axis=1)
    t1 = np.concatenate([t, np.ones((B, 1), np.float32)], axis=1)
    grid = sg.n_ctas(B)
    part = np.zeros((grid, S, d + 1), np.float32)
    for grp in range(-(-B // 8)):
        k = grp % grid
        acc = part[k] if grp >= grid and mutant != "cta_overwrite" else np.zeros((S, d + 1), np.float32)
        for i in range(grp * 8, min(B, grp * 8 + 8)):
            acc = sg.fma32(h[i][:, None], t1[i][None, :], acc)
        part[k] = acc
    gc_neg = part[0]
    for k in range(1, grid):
        gc_neg = gc_neg + part[k]
    sp = lambda v: (np.maximum(v.astype(np.float64), 0) + np.log1p(np.exp(-np.abs(v.astype(np.float64))))).astype(np.float32)  # noqa
    row = sp(-x)
    for j in range(S):
        row = row + sp(xn[:, j])
    lanes = np.zeros(32, np.float32)
    for i in range(B):
        lanes[i % 32] = lanes[i % 32] + row[i]
    loss = sg.butterfly(lanes) / fB
    return dict(loss=loss, aff=aff, neg_aff=neg_aff, gt=gt, gc_pos=gc_pos, gc_neg=gc_neg)


def _bits_equal(a, b):
    a, b = np.ascontiguousarray(a, np.float32), np.ascontiguousarray(b, np.float32)
    return a.shape == b.shape and a.tobytes() == b.tobytes()


# ---------------------------------------------------------------------------------------------------- the emulation passes
@pytest.mark.parametrize("d", EMBED_D)
def test_embed_emulation_passes(d):
    n_rows, lists = embed_case(d)
    assert _bits_equal(emulate_embed(lists, n_rows, d), sg.embedding_grad_reference(lists, n_rows, d))
    n_rows, lists = embed_case(d, seed=1)
    sites = embed_sites(lists)
    assert _bits_equal(emulate_embed(lists, n_rows, d, sites), sg.embedding_grad_reference(lists, n_rows, d, sites))


def test_embed_emulation_passes_on_the_reddit_shape():
    n_rows, d, lists = reddit_case()
    assert _bits_equal(emulate_embed(lists, n_rows, d), sg.embedding_grad_reference(lists, n_rows, d))


@pytest.mark.parametrize("lr", [0.05, 0.3])
@pytest.mark.parametrize("d", [1, 51, 257])
def test_sgd_emulation_passes(d, lr):
    table, lists = sgd_case(d)
    alpha = float(_f32(-lr))
    got = emulate_embed(lists, table.shape[0], d, table=table, alpha=alpha)
    assert got.tobytes() == sg.embedding_sgd_reference(table, lists, alpha, d).tobytes()


@pytest.mark.parametrize("B, S, d", SG_CASES, ids=["B%d_S%d_d%d" % c for c in SG_CASES])
def test_skipgram_emulation_passes(B, S, d):
    T, C, b1, b2, neg = sg_case(B, S, d)
    fails, stats = sg.check_skipgram(T, C, d, b1, b2, neg, emulate_skipgram(T, C, d, b1, b2, neg))
    assert not fails, (fails, stats)
    if B >= 512:                                                   # the GPU file asserts this on the kernel's aff
        t, c, b, _, _ = sg.skipgram_operands(T, C, d, b1, b2, neg)
        x = sg.lane_dot(t, c) + b
        assert (x > 20).any() and (x < -20).any()


# ---------------------------------------------------------------------------------------------------- each mutant fails
MUTANT_D = 257          # three column tiles at the SGD shape; the grad shapes use 129 (two tiles, a 60,000-entry hub)


@pytest.mark.parametrize("mutant", sorted(EMBED_MUTANTS))
def test_each_embed_mutant_fails_a_check(mutant):
    kind = EMBED_MUTANTS[mutant]
    if kind == "sgd":
        table, lists = sgd_case(MUTANT_D)
        alpha = float(_f32(-0.05))
        got = emulate_embed(lists, table.shape[0], MUTANT_D, table=table, alpha=alpha, mutant=mutant)
        assert got.tobytes() != sg.embedding_sgd_reference(table, lists, alpha, MUTANT_D).tobytes(), mutant
        return
    d = 129
    n_rows, lists = embed_case(d, seed=1 if kind == "dropout" else 0)
    sites = embed_sites(lists) if kind == "dropout" else None
    with np.errstate(invalid="ignore"):
        got = emulate_embed(lists, n_rows, d, sites, mutant=mutant)
    assert not _bits_equal(got, sg.embedding_grad_reference(lists, n_rows, d, sites)), mutant


@pytest.mark.parametrize("mutant", SG_MUTANTS)
def test_each_skipgram_mutant_fails_a_check(mutant):
    B, S, d = 2049, 20, 50
    T, C, b1, b2, neg = sg_case(B, S, d)
    fails, stats = sg.check_skipgram(T, C, d, b1, b2, neg, emulate_skipgram(T, C, d, b1, b2, neg, mutant))
    assert fails, (mutant, stats)
    print(mutant, "fails", fails)
